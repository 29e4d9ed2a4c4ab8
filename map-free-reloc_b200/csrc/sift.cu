// SIFT detector + descriptor engine for B uint8 gray images of one size: OpenCV 4.x
// cv2.SIFT_create(nfeatures).detectAndCompute at the default settings (3 layers per octave, contrast threshold 0.04,
// edge threshold 10, sigma 1.6, first octave -1, CV_32F descriptors), the detector of the reference's SIFT plugins
// (lib/models/matching/feature_matching.py:53-118, etc/feature_matching_baselines/matchers.py:123-188).
//
// One static launch list, no host synchronisation inside: every count-dependent stage reads its extent from device
// counters, so detect() can be replayed as a CUDA graph. Stages:
//   pyramid      u8 -> float x2 bilinear (resize_linear's float path), Gaussian cascade with getGaussianKernel(CV_32F)
//                coefficients and BORDER_REFLECT_101, row + column pass fused through a shared-memory tile that also
//                writes the DoG level; next octave = every other pixel of level 3
//   extrema      thread per pixel of DoG layers 1..3: 26-neighbour test + adjustLocalExtrema, appended through a counter
//   orientation  warp per extremum: 36-bin histogram (fastAtan2), [1 4 6 4 1]/16 smoothing, every peak >= 0.8 max
//   selection    block per image: sort by (response desc, x, y, size, angle, octave), drop exact duplicates,
//                retainBest(nfeatures) (every keypoint with response >= the N-th), rescale to input pixels
//   descriptors  block per keypoint: 4x4x8 histogram, trilinear weights, clamp 0.2, x512, saturate to uchar
// Determinism: the atomic append order never reaches an output. Selection sorts on a total order, and every
// histogram bin is summed by one thread in the raster order of its window (OpenCV's order), never with float atomics.
// Compiled with -fmad=false so that float expressions round operation by operation as OpenCV's scalar code writes
// them; the fused operations of OpenCV's SIMD paths (fastAtan2, magnitude, smoothing) are written as fmaf.
#include "sift.cuh"

#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <vector>

#include "descriptor_match.cuh"
#include "engine_core.cuh"

namespace mfr {

int resize_linear(const void* src, int src_is_u8, int sw, int sh, long long src_stride, int channels, float* dst, int dw, int dh,
                  int mode, float out_scale, int chw, cudaStream_t st);   // image_io.cu

namespace {

constexpr int kLayers = 3;            // nOctaveLayers
constexpr int kLevels = kLayers + 3;  // Gaussian levels per octave
constexpr int kDogs = kLayers + 2;    // DoG levels per octave
constexpr int kBorder = 5;            // SIFT_IMG_BORDER
constexpr int kMaxOct = 16;
constexpr int kMaxR = 16;             // largest blur radius (ksize 33); the cascade needs 13
constexpr int kOriBins = 36;
constexpr int kOriMaxR = 16;          // cvRound(4.5 * 1.6 * 2^(3.5/3)) = 16
constexpr int kOriMaxS = (2 * kOriMaxR + 1) * (2 * kOriMaxR + 1);
constexpr int kD = 4, kN = 8;
constexpr int kHistLen = (kD + 2) * (kD + 2) * (kN + 2);   // 360

struct Kernel1D { float c[2 * kMaxR + 1]; int r; };
struct Pyr { const float* g[kMaxOct]; int h[kMaxOct], w[kMaxOct]; int n; };

__device__ __forceinline__ int reflect101(int p, int len) {   // borderInterpolate(BORDER_REFLECT_101)
  if (len == 1) return 0;
  while (static_cast<unsigned>(p) >= static_cast<unsigned>(len)) p = p < 0 ? -p : 2 * len - 2 - p;
  return p;
}

// cv::hal::fastAtan2 in degrees, the SIMD form (v_fma polynomial)
__device__ __forceinline__ float fast_atan2(float y, float x) {
  const float p1 = 0.9997878412794807f * 57.295779513082320876798f, p3 = -0.3258083974640975f * 57.295779513082320876798f;
  const float p5 = 0.1555786518463281f * 57.295779513082320876798f, p7 = -0.04432655554792128f * 57.295779513082320876798f;
  const float ax = fabsf(x), ay = fabsf(y);
  const float c = fminf(ax, ay) / (fmaxf(ax, ay) + static_cast<float>(DBL_EPSILON));
  const float cc = c * c;
  float a = fmaf(fmaf(fmaf(cc, p7, p5), cc, p3), cc, p1) * c;
  if (!(ax >= ay)) a = 90.f - a;
  if (x < 0.f) a = 180.f - a;
  if (y < 0.f) a = 360.f - a;
  return a;
}

// ---------------------------------------------------------------------------------------------------- pyramid
constexpr int kTile = 32;
// dst = GaussianBlur(src) for every image (blockIdx.z); dog (optional) = dst - src
__global__ void __launch_bounds__(256) blur_kernel(const float* __restrict__ src, long long src_img, float* __restrict__ dst,
                                                   long long dst_img, float* __restrict__ dog, long long dog_img, int h, int w,
                                                   Kernel1D k) {
  __shared__ float s_in[(kTile + 2 * kMaxR) * (kTile + 2 * kMaxR)];
  __shared__ float s_mid[(kTile + 2 * kMaxR) * kTile];
  const int r = k.r, tw = kTile + 2 * r, th = kTile + 2 * r;
  const int x0 = blockIdx.x * kTile, y0 = blockIdx.y * kTile, b = blockIdx.z;
  const float* S = src + b * src_img;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
  for (int i = tid; i < tw * th; i += nt) {
    const int ly = i / tw, lx = i - ly * tw;
    s_in[i] = S[static_cast<size_t>(reflect101(y0 - r + ly, h)) * w + reflect101(x0 - r + lx, w)];
  }
  __syncthreads();
  for (int i = tid; i < th * kTile; i += nt) {   // row filter
    const int ly = i / kTile, lx = i - ly * kTile;
    const float* p = s_in + ly * tw + lx;
    float s = 0.f;
    for (int j = 0; j <= 2 * r; ++j) s += k.c[j] * p[j];
    s_mid[i] = s;
  }
  __syncthreads();
  for (int i = tid; i < kTile * kTile; i += nt) {   // column filter
    const int ly = i / kTile, lx = i - ly * kTile;
    const int y = y0 + ly, x = x0 + lx;
    if (y >= h || x >= w) continue;
    float s = 0.f;
    for (int j = 0; j <= 2 * r; ++j) s += k.c[j] * s_mid[(ly + j) * kTile + lx];
    const size_t o = static_cast<size_t>(y) * w + x;
    dst[b * dst_img + o] = s;
    if (dog) dog[b * dog_img + o] = s - s_in[(ly + r) * tw + lx + r];
  }
}

// next octave's base: resize(INTER_NEAREST) of level 3 to (w/2, h/2) = every other pixel
__global__ void downsample_kernel(const float* __restrict__ src, long long src_img, int sw, float* __restrict__ dst,
                                  long long dst_img, int h, int w) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (x >= w) return;
  dst[b * dst_img + static_cast<size_t>(y) * w + x] = src[b * src_img + static_cast<size_t>(2 * y) * sw + 2 * x];
}

// ---------------------------------------------------------------------------------------------------- extrema
// Matx33f::solve(DECOMP_LU) for one right-hand side in OpenCV 4.x: Cramer's rule in float (Matx_FastSolveOp<float,3,1>)
__device__ __forceinline__ void solve3(const float a[3][3], const float b[3], float x[3]) {
  const float det = a[0][0] * (a[1][1] * a[2][2] - a[2][1] * a[1][2]) - a[0][1] * (a[1][0] * a[2][2] - a[2][0] * a[1][2]) +
                    a[0][2] * (a[1][0] * a[2][1] - a[2][0] * a[1][1]);
  if (det == 0.f) { x[0] = x[1] = x[2] = 0.f; return; }
  const float d = 1.f / det;
  x[0] = d * (b[0] * (a[1][1] * a[2][2] - a[1][2] * a[2][1]) - a[0][1] * (b[1] * a[2][2] - a[1][2] * b[2]) +
              a[0][2] * (b[1] * a[2][1] - a[1][1] * b[2]));
  x[1] = d * (a[0][0] * (b[1] * a[2][2] - a[1][2] * b[2]) - b[0] * (a[1][0] * a[2][2] - a[1][2] * a[2][0]) +
              a[0][2] * (a[1][0] * b[2] - b[1] * a[2][0]));
  x[2] = d * (a[0][0] * (a[1][1] * b[2] - b[1] * a[2][1]) - a[0][1] * (a[1][0] * b[2] - b[1] * a[2][0]) +
              b[0] * (a[1][0] * a[2][1] - a[1][1] * a[2][0]));
}

// thread per pixel of DoG layers 1..3 (blockIdx.z = image * 3 + layer - 1): findScaleSpaceExtrema + adjustLocalExtrema
__global__ void __launch_bounds__(256) extrema_kernel(const float* __restrict__ dog, int h, int w, int o, int cap,
                                                      int* __restrict__ count, float4* __restrict__ ext_f,
                                                      int4* __restrict__ ext_i) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int b = blockIdx.z / kLayers, layer0 = blockIdx.z % kLayers + 1;
  if (x < kBorder || x >= w - kBorder || y < kBorder || y >= h - kBorder) return;
  const size_t plane = static_cast<size_t>(h) * w;
  const float* D = dog + static_cast<size_t>(b) * kDogs * plane;
  auto at = [&](int l, int rr, int cc) { return D[l * plane + static_cast<size_t>(rr) * w + cc]; };
  const float v = at(layer0, y, x);
  if (!(fabsf(v) > 1.f)) return;   // cvFloor(0.5 * 0.04 / 3 * 255) = 1
  bool ok = true;
  for (int l = layer0 - 1; l <= layer0 + 1 && ok; ++l)
    for (int dy = -1; dy <= 1 && ok; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const float n = at(l, y + dy, x + dx);
        if (v > 0.f ? !(v >= n) : !(v <= n)) { ok = false; break; }
      }
  if (!ok) return;
  const float img_scale = 1.f / 255.f, deriv_scale = img_scale * 0.5f, cross_scale = img_scale * 0.25f;
  int layer = layer0, r = y, c = x, i = 0;
  float xi = 0.f, xr = 0.f, xc = 0.f;
  for (; i < 5; ++i) {
    const float dD[3] = {(at(layer, r, c + 1) - at(layer, r, c - 1)) * deriv_scale,
                         (at(layer, r + 1, c) - at(layer, r - 1, c)) * deriv_scale,
                         (at(layer + 1, r, c) - at(layer - 1, r, c)) * deriv_scale};
    const float v2 = at(layer, r, c) * 2.f;
    const float dxx = (at(layer, r, c + 1) + at(layer, r, c - 1) - v2) * img_scale;
    const float dyy = (at(layer, r + 1, c) + at(layer, r - 1, c) - v2) * img_scale;
    const float dss = (at(layer + 1, r, c) + at(layer - 1, r, c) - v2) * img_scale;
    const float dxy = (at(layer, r + 1, c + 1) - at(layer, r + 1, c - 1) - at(layer, r - 1, c + 1) + at(layer, r - 1, c - 1)) * cross_scale;
    const float dxs = (at(layer + 1, r, c + 1) - at(layer + 1, r, c - 1) - at(layer - 1, r, c + 1) + at(layer - 1, r, c - 1)) * cross_scale;
    const float dys = (at(layer + 1, r + 1, c) - at(layer + 1, r - 1, c) - at(layer - 1, r + 1, c) + at(layer - 1, r - 1, c)) * cross_scale;
    const float H[3][3] = {{dxx, dxy, dxs}, {dxy, dyy, dys}, {dxs, dys, dss}};
    float X[3];
    solve3(H, dD, X);
    xi = -X[2]; xr = -X[1]; xc = -X[0];
    if (fabsf(xi) < 0.5f && fabsf(xr) < 0.5f && fabsf(xc) < 0.5f) break;
    const float big = static_cast<float>(INT_MAX / 3);
    if (fabsf(xi) > big || fabsf(xr) > big || fabsf(xc) > big) return;
    c += __float2int_rn(xc); r += __float2int_rn(xr); layer += __float2int_rn(xi);
    if (layer < 1 || layer > kLayers || c < kBorder || c >= w - kBorder || r < kBorder || r >= h - kBorder) return;
  }
  if (i >= 5) return;
  const float dD0 = (at(layer, r, c + 1) - at(layer, r, c - 1)) * deriv_scale;
  const float dD1 = (at(layer, r + 1, c) - at(layer, r - 1, c)) * deriv_scale;
  const float dD2 = (at(layer + 1, r, c) - at(layer - 1, r, c)) * deriv_scale;
  float t = 0.f;
  t = t + dD0 * xc; t = t + dD1 * xr; t = t + dD2 * xi;
  const float contr = at(layer, r, c) * img_scale + t * 0.5f;
  if (fabsf(contr) * static_cast<float>(kLayers) < 0.04f) return;
  const float v2 = at(layer, r, c) * 2.f;
  const float dxx = (at(layer, r, c + 1) + at(layer, r, c - 1) - v2) * img_scale;
  const float dyy = (at(layer, r + 1, c) + at(layer, r - 1, c) - v2) * img_scale;
  const float dxy = (at(layer, r + 1, c + 1) - at(layer, r + 1, c - 1) - at(layer, r - 1, c + 1) + at(layer, r - 1, c - 1)) * cross_scale;
  const float tr = dxx + dyy, det = dxx * dyy - dxy * dxy;
  if (det <= 0.f || tr * tr * 10.f >= 121.f * det) return;
  const float s = static_cast<float>(1 << o);
  const float4 f = make_float4((static_cast<float>(c) + xc) * s, (static_cast<float>(r) + xr) * s,
                               1.6f * powf(2.f, (static_cast<float>(layer) + xi) / static_cast<float>(kLayers)) * s * 2.f,
                               fabsf(contr));
  const int oct = o + (layer << 8) + (__double2int_rn((static_cast<double>(xi) + 0.5) * 255.0) << 16);
  const int slot = atomicAdd(count + b, 1);
  if (slot < cap) {
    ext_f[static_cast<size_t>(b) * cap + slot] = f;
    ext_i[static_cast<size_t>(b) * cap + slot] = make_int4(oct, layer, r, c);
  }
}

// ---------------------------------------------------------------------------------------------------- orientation
constexpr int kOriWarps = 4;
// warp per extremum (grid-stride, blockIdx.y = image): calcOrientationHist + the peak loop of findScaleSpaceExtrema
__global__ void __launch_bounds__(kOriWarps * 32) orientation_kernel(Pyr pyr, const int* __restrict__ ext_count,
                                                                     const float4* __restrict__ ext_f,
                                                                     const int4* __restrict__ ext_i, int cap,
                                                                     int* __restrict__ kp_count, float* __restrict__ kp,
                                                                     int* __restrict__ kp_oct) {
  __shared__ int s_bin[kOriWarps][kOriMaxS];
  __shared__ float s_val[kOriWarps][kOriMaxS];
  __shared__ float s_hist[kOriWarps][kOriBins + 4];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
  const int n = min(ext_count[b], cap);
  for (int e = blockIdx.x * kOriWarps + warp; e < n; e += gridDim.x * kOriWarps) {
    const float4 f = ext_f[static_cast<size_t>(b) * cap + e];
    const int4 id = ext_i[static_cast<size_t>(b) * cap + e];
    const int o = id.x & 255, layer = id.y, pr = id.z, pc = id.w;
    const int h = pyr.h[o], w = pyr.w[o];
    const float* img = pyr.g[o] + (static_cast<size_t>(b) * kLevels + layer) * h * w;
    const float scl = f.z * 0.5f / static_cast<float>(1 << o);
    const int rad = min(__float2int_rn(4.5f * scl), kOriMaxR);
    const float sigma = 1.5f * scl;
    const float escale = -1.f / (2.f * sigma * sigma);
    const int side = 2 * rad + 1, len = side * side;
    for (int k = lane; k < len; k += 32) {
      const int i = k / side - rad, j = k % side - rad;
      const int yy = pr + i, xx = pc + j;
      int bin = -1; float val = 0.f;
      if (yy > 0 && yy < h - 1 && xx > 0 && xx < w - 1) {
        const float dx = img[static_cast<size_t>(yy) * w + xx + 1] - img[static_cast<size_t>(yy) * w + xx - 1];
        const float dy = img[static_cast<size_t>(yy - 1) * w + xx] - img[static_cast<size_t>(yy + 1) * w + xx];
        const float wt = expf(static_cast<float>(i * i + j * j) * escale);
        const float ori = fast_atan2(dy, dx);
        const float mag = sqrtf(fmaf(dx, dx, dy * dy));
        bin = __float2int_rn((static_cast<float>(kOriBins) / 360.f) * ori);
        if (bin >= kOriBins) bin -= kOriBins;
        if (bin < 0) bin += kOriBins;
        val = wt * mag;
      }
      s_bin[warp][k] = bin; s_val[warp][k] = val;
    }
    __syncwarp();
    float h0 = 0.f, h1 = 0.f;   // lane owns bins lane and lane + 32, summed in raster order
    for (int k = 0; k < len; ++k) {
      const int bin = s_bin[warp][k];
      if (bin == lane) h0 += s_val[warp][k];
      if (bin == lane + 32) h1 += s_val[warp][k];
    }
    float* t = s_hist[warp] + 2;   // t[-2 .. 37]
    t[lane] = h0;
    if (lane < kOriBins - 32) t[lane + 32] = h1;
    __syncwarp();
    if (lane < 2) { t[-1 - lane] = t[kOriBins - 1 - lane]; t[kOriBins + lane] = t[lane]; }
    __syncwarp();
    float sm0 = fmaf(t[lane - 2] + t[lane + 2], 1.f / 16.f, fmaf(t[lane - 1] + t[lane + 1], 4.f / 16.f, t[lane] * (6.f / 16.f)));
    float sm1 = -1.f;
    if (lane < kOriBins - 32) {
      const int q = lane + 32;
      sm1 = fmaf(t[q - 2] + t[q + 2], 1.f / 16.f, fmaf(t[q - 1] + t[q + 1], 4.f / 16.f, t[q] * (6.f / 16.f)));
    }
    __syncwarp();
    float* hs = s_hist[warp];
    hs[lane] = sm0;
    if (lane < kOriBins - 32) hs[lane + 32] = sm1;
    __syncwarp();
    if (lane == 0) {
      float omax = hs[0];
      for (int j = 1; j < kOriBins; ++j) omax = fmaxf(omax, hs[j]);
      const float thr = omax * 0.8f;
      for (int j = 0; j < kOriBins; ++j) {
        const int l = j > 0 ? j - 1 : kOriBins - 1, r2 = j < kOriBins - 1 ? j + 1 : 0;
        if (hs[j] > hs[l] && hs[j] > hs[r2] && hs[j] >= thr) {
          float bin = static_cast<float>(j) + 0.5f * (hs[l] - hs[r2]) / (hs[l] - 2.f * hs[j] + hs[r2]);
          bin = bin < 0.f ? static_cast<float>(kOriBins) + bin : bin >= static_cast<float>(kOriBins) ? bin - static_cast<float>(kOriBins) : bin;
          float angle = 360.f - (360.f / kOriBins) * bin;
          if (fabsf(angle - 360.f) < FLT_EPSILON) angle = 0.f;
          const int slot = atomicAdd(kp_count + b, 1);
          if (slot < cap) {
            float* q = kp + (static_cast<size_t>(b) * cap + slot) * 5;
            q[0] = f.x; q[1] = f.y; q[2] = f.z; q[3] = angle; q[4] = f.w;
            kp_oct[static_cast<size_t>(b) * cap + slot] = id.x;
          }
        }
      }
    }
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------- selection
// total order: response descending, then x, y, size, angle, octave ascending
__device__ __forceinline__ bool kp_before(const float* a, int oa, const float* b, int ob) {
  if (a[4] != b[4]) return a[4] > b[4];
  for (int k = 0; k < 4; ++k)
    if (a[k] != b[k]) return a[k] < b[k];
  return oa < ob;
}

constexpr int kSelThreads = 1024;
// block per image: sort (bitonic on a 64-bit (response desc, x) key, then the full order inside equal keys),
// removeDuplicatedSorted, retainBest, rescale to input pixels (firstOctave = -1), gather
__global__ void __launch_bounds__(kSelThreads) select_kernel(const int* __restrict__ kp_count, const float* __restrict__ kp,
                                                             const int* __restrict__ kp_oct, int cap, int cap2,
                                                             unsigned long long* __restrict__ keys, int* __restrict__ idx,
                                                             int* __restrict__ rank, int nfeatures, int* __restrict__ out_count,
                                                             float* __restrict__ out_kp, int* __restrict__ out_oct) {
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = min(kp_count[b], cap);
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  unsigned long long* K = keys + static_cast<size_t>(b) * cap2;
  int* I = idx + static_cast<size_t>(b) * cap2;
  int* Rk = rank + static_cast<size_t>(b) * cap;
  const float* P = kp + static_cast<size_t>(b) * cap * 5;
  const int* O = kp_oct + static_cast<size_t>(b) * cap;
  for (int i = tid; i < n2; i += kSelThreads) {
    if (i < n) {
      K[i] = (static_cast<unsigned long long>(~__float_as_uint(P[i * 5 + 4])) << 32) | __float_as_uint(P[i * 5]);
      I[i] = i;
    } else {
      K[i] = ~0ull; I[i] = -1;
    }
  }
  __syncthreads();
  for (int k = 2; k <= n2; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < n2; i += kSelThreads) {
        const int l = i ^ j;
        if (l > i) {
          const unsigned long long a = K[i], c = K[l];
          const bool up = (i & k) == 0;
          if ((a > c) == up && a != c) { K[i] = c; K[l] = a; const int t = I[i]; I[i] = I[l]; I[l] = t; }
        }
      }
      __syncthreads();
    }
  // runs of equal keys (the orientations of one point share response and x): insertion sort on the full order
  for (int i = tid; i < n; i += kSelThreads) {
    if (i > 0 && K[i - 1] == K[i]) continue;
    int e = i + 1;
    while (e < n && K[e] == K[i]) ++e;
    for (int a = i + 1; a < e; ++a) {
      const int v = I[a];
      int q = a - 1;
      while (q >= i && kp_before(P + v * 5, O[v], P + I[q] * 5, O[I[q]])) { I[q + 1] = I[q]; --q; }
      I[q + 1] = v;
    }
  }
  __syncthreads();
  // duplicates (same pt, size, angle as the previous keypoint) and the rank of every kept one
  __shared__ int s_warp[kSelThreads / 32];
  __shared__ int s_base, s_cut_set;
  __shared__ float s_cut;
  if (tid == 0) { s_base = 0; s_cut_set = 0; }
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += kSelThreads) {
    const int i = c0 + tid;
    int keep = 0;
    if (i < n) {
      const float* a = P + I[i] * 5;
      keep = 1;
      if (i > 0) {
        const float* p = P + I[i - 1] * 5;
        keep = !(a[0] == p[0] && a[1] == p[1] && a[2] == p[2] && a[3] == p[3]);
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    const int lane = tid & 31, wid = tid >> 5;
    if (lane == 0) s_warp[wid] = __popc(m);
    __syncthreads();
    if (tid == 0) {
      int s = s_base;
      for (int w2 = 0; w2 < kSelThreads / 32; ++w2) { const int t = s_warp[w2]; s_warp[w2] = s; s += t; }
      s_base = s;
    }
    __syncthreads();
    if (i < n) {
      const int rk = keep ? s_warp[wid] + __popc(m & ((1u << lane) - 1u)) : -1;
      Rk[i] = rk;
      if (rk == nfeatures - 1 && nfeatures > 0) { s_cut = P[I[i] * 5 + 4]; s_cut_set = 1; }
    }
    __syncthreads();
  }
  const int total = s_base;
  const bool limit = nfeatures > 0 && total > nfeatures && s_cut_set;
  const float cut = s_cut;
  __shared__ int s_count;
  if (tid == 0) s_count = 0;
  __syncthreads();
  int local = 0;
  for (int i = tid; i < n; i += kSelThreads) {
    const int rk = Rk[i];
    if (rk < 0) continue;
    const float* a = P + I[i] * 5;
    if (limit && !(a[4] >= cut)) continue;
    float* q = out_kp + (static_cast<size_t>(b) * cap + rk) * 5;
    q[0] = a[0] * 0.5f; q[1] = a[1] * 0.5f; q[2] = a[2] * 0.5f; q[3] = a[3]; q[4] = a[4];
    const int oc = O[I[i]];
    out_oct[static_cast<size_t>(b) * cap + rk] = (oc & ~255) | ((oc - 1) & 255);
    local = max(local, rk + 1);
  }
  atomicMax(&s_count, local);
  __syncthreads();
  if (tid == 0) out_count[b] = s_count;
}

// ---------------------------------------------------------------------------------------------------- descriptors
constexpr int kDescThreads = 256;
// block per keypoint (grid-stride, blockIdx.y = image): calcSIFTDescriptor on the keypoint's Gaussian level
__global__ void __launch_bounds__(kDescThreads) descriptor_kernel(Pyr pyr, const int* __restrict__ count,
                                                                  const float* __restrict__ kps, const int* __restrict__ octs,
                                                                  int cap, int root, float* __restrict__ desc) {
  __shared__ int s_idx[kDescThreads];
  __shared__ float s_v[kDescThreads][8];
  __shared__ float s_hist[kHistLen];
  __shared__ float s_dst[128];
  __shared__ double s_red[4];
  const int b = blockIdx.y, tid = threadIdx.x;
  const int n = count[b];
  constexpr int C = kN + 2, R = (kD + 2) * (kN + 2);   // the 8 corners of a sample: idx + (z & 1) + C (z >> 1 & 1) + R (z >> 2)
  for (int kpi = blockIdx.x; kpi < n; kpi += gridDim.x) {
    const float* kp = kps + (static_cast<size_t>(b) * cap + kpi) * 5;
    const int oc = octs[static_cast<size_t>(b) * cap + kpi];
    int octave = oc & 255;
    const int layer = (oc >> 8) & 255;
    octave = octave < 128 ? octave : (-128 | octave);
    const float scale = octave >= 0 ? 1.f / static_cast<float>(1 << octave) : static_cast<float>(1 << -octave);
    const int o = octave + 1;
    const int h = pyr.h[o], w = pyr.w[o];
    const float* img = pyr.g[o] + (static_cast<size_t>(b) * kLevels + layer) * h * w;
    const float size = kp[2] * scale, ptx = kp[0] * scale, pty = kp[1] * scale;
    float ori = 360.f - kp[3];
    if (fabsf(ori - 360.f) < FLT_EPSILON) ori = 0.f;
    const float scl = size * 0.5f;
    const int px = __float2int_rn(ptx), py = __float2int_rn(pty);
    float cos_t = cosf(ori * static_cast<float>(3.14159265358979323846 / 180));
    float sin_t = sinf(ori * static_cast<float>(3.14159265358979323846 / 180));
    const float bins_per_rad = kN / 360.f, exp_scale = -1.f / (kD * kD * 0.5f);
    const float hist_width = 3.f * scl;
    int rad = __float2int_rn(hist_width * 1.4142135623730951f * static_cast<float>(kD + 1) * 0.5f);
    rad = min(rad, static_cast<int>(sqrt(static_cast<double>(w) * w + static_cast<double>(h) * h)));
    cos_t /= hist_width; sin_t /= hist_width;
    const int side = 2 * rad + 1, len = side * side;
    float hb0 = 0.f, hb1 = 0.f;   // this thread's bins: tid and tid + 256
    for (int c0 = 0; c0 < len; c0 += kDescThreads) {
      const int k = c0 + tid;
      int id = INT_MIN / 2;
      if (k < len) {
        const int i = k / side - rad, j = k % side - rad;
        const float c_rot = static_cast<float>(j) * cos_t - static_cast<float>(i) * sin_t;
        const float r_rot = static_cast<float>(j) * sin_t + static_cast<float>(i) * cos_t;
        float rbin = r_rot + static_cast<float>(kD / 2) - 0.5f;
        float cbin = c_rot + static_cast<float>(kD / 2) - 0.5f;
        const int r = py + i, c = px + j;
        if (rbin > -1.f && rbin < kD && cbin > -1.f && cbin < kD && r > 0 && r < h - 1 && c > 0 && c < w - 1) {
          const float dx = img[static_cast<size_t>(r) * w + c + 1] - img[static_cast<size_t>(r) * w + c - 1];
          const float dy = img[static_cast<size_t>(r - 1) * w + c] - img[static_cast<size_t>(r + 1) * w + c];
          const float wt = expf((c_rot * c_rot + r_rot * r_rot) * exp_scale);
          const float mag = sqrtf(fmaf(dx, dx, dy * dy)) * wt;
          float obin = (fast_atan2(dy, dx) - ori) * bins_per_rad;
          const int r0 = static_cast<int>(floorf(rbin)), cb0 = static_cast<int>(floorf(cbin));
          int o0 = static_cast<int>(floorf(obin));
          rbin -= static_cast<float>(r0); cbin -= static_cast<float>(cb0); obin -= static_cast<float>(o0);
          if (o0 < 0) o0 += kN;
          if (o0 >= kN) o0 -= kN;
          const float v_r1 = mag * rbin, v_r0 = mag - v_r1;
          const float v_rc11 = v_r1 * cbin, v_rc10 = v_r1 - v_rc11;
          const float v_rc01 = v_r0 * cbin, v_rc00 = v_r0 - v_rc01;
          const float v111 = v_rc11 * obin, v110 = v_rc11 - v111;
          const float v101 = v_rc10 * obin, v100 = v_rc10 - v101;
          const float v011 = v_rc01 * obin, v010 = v_rc01 - v011;
          const float v001 = v_rc00 * obin, v000 = v_rc00 - v001;
          id = ((r0 + 1) * (kD + 2) + cb0 + 1) * (kN + 2) + o0;
          float* sv = s_v[tid];
          sv[0] = v000; sv[1] = v001; sv[2] = v010; sv[3] = v011; sv[4] = v100; sv[5] = v101; sv[6] = v110; sv[7] = v111;
        }
      }
      s_idx[tid] = id;
      __syncthreads();
      const int m = min(kDescThreads, len - c0);
      for (int q = 0; q < m; ++q) {   // raster order: OpenCV's summation order for every bin
        const int base = s_idx[q];
        const int d0 = tid - base, d1 = tid + kDescThreads - base;
#pragma unroll
        for (int z = 0; z < 8; ++z) {
          const int off = (z & 1) + ((z >> 1) & 1) * C + (z >> 2) * R;
          if (d0 == off) hb0 += s_v[q][z];
          if (d1 == off) hb1 += s_v[q][z];
        }
      }
      __syncthreads();
    }
    s_hist[tid] = hb0;
    if (tid + kDescThreads < kHistLen) s_hist[tid + kDescThreads] = hb1;
    __syncthreads();
    double sq = 0.0;
    if (tid < 128) {
      const int i = tid >> 5, j = (tid >> 3) & 3, k = tid & 7;
      const int idx = ((i + 1) * (kD + 2) + (j + 1)) * (kN + 2);
      const float v = k < 2 ? s_hist[idx + k] + s_hist[idx + kN + k] : s_hist[idx + k];
      s_dst[tid] = v;
      sq = static_cast<double>(v) * v;
    }
    for (int s = 16; s > 0; s >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, s);
    if (tid < 128 && (tid & 31) == 0) s_red[tid >> 5] = sq;
    __syncthreads();
    const float nrm1 = static_cast<float>(s_red[0] + s_red[1] + s_red[2] + s_red[3]);
    const float thr = sqrtf(nrm1) * 0.2f;
    float val = 0.f;
    sq = 0.0;
    if (tid < 128) { val = fminf(s_dst[tid], thr); sq = static_cast<double>(val) * val; }
    __syncthreads();
    for (int s = 16; s > 0; s >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, s);
    if (tid < 128 && (tid & 31) == 0) s_red[tid >> 5] = sq;
    __syncthreads();
    const float nrm2 = 512.f / fmaxf(sqrtf(static_cast<float>(s_red[0] + s_red[1] + s_red[2] + s_red[3])), FLT_EPSILON);
    float u = 0.f;
    if (tid < 128) u = fminf(fmaxf(rintf(val * nrm2), 0.f), 255.f);   // saturate_cast<uchar>
    if (root) {   // RootSIFT: L1 normalisation (eps 1e-7), square root; the sum of integers is exact in any order
      __syncthreads();
      double l1 = tid < 128 ? u : 0.0;
      for (int s = 16; s > 0; s >>= 1) l1 += __shfl_xor_sync(0xffffffffu, l1, s);
      if (tid < 128 && (tid & 31) == 0) s_red[tid >> 5] = l1;
      __syncthreads();
      const float l1f = static_cast<float>(s_red[0] + s_red[1] + s_red[2] + s_red[3]);
      u = sqrtf(u / (l1f + 1e-7f));
    }
    if (tid < 128) desc[(static_cast<size_t>(b) * cap + kpi) * 128 + tid] = u;
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------- ratio test
// block per pair: good[q] = (train count >= 2) && d1 < ratio * d2; pair_n[p] = number of good queries. Pair p's query /
// train counts are qc[p * qs] / tc[p * ts].
__global__ void ratio_count_kernel(const int* __restrict__ qc, int qs, const int* __restrict__ tc, int ts,
                                   const float* __restrict__ d1, const float* __restrict__ d2, int cap, float ratio,
                                   unsigned char* __restrict__ good, int* __restrict__ pair_n) {
  const int p = blockIdx.x;
  const int nq = qc[p * qs], nt = tc[p * ts];
  __shared__ int s_n;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  int local = 0;
  for (int q = threadIdx.x; q < nq; q += blockDim.x) {
    const size_t o = static_cast<size_t>(p) * cap + q;
    const bool g = nt >= 2 && d1[o] < ratio * d2[o];
    good[o] = g;
    local += g;
  }
  atomicAdd(&s_n, local);
  __syncthreads();
  if (threadIdx.x == 0) pair_n[p] = s_n;
}

__global__ void pair_offsets_kernel(const int* __restrict__ pair_n, int P, int* __restrict__ offsets) {
  if (threadIdx.x != 0) return;
  int s = 0;
  for (int p = 0; p < P; ++p) { offsets[p] = s; s += pair_n[p]; }
  offsets[P] = s;
}

// block per pair: ordered compaction of the good queries (query order, = np.where(good)) into the pose back end's layout.
// Pair p's query keypoints are image p * s0 of kp0 (qc[p * qs] of them), its train keypoints image p * s1 of kp1.
__global__ void __launch_bounds__(256) compact_matches_kernel(const int* __restrict__ qc, int qs, const unsigned char* __restrict__ good,
                                                              const int* __restrict__ i1, const float* __restrict__ kp0, int s0,
                                                              const float* __restrict__ kp1, int s1, int cap,
                                                              const int* __restrict__ offsets, float* __restrict__ k0,
                                                              float* __restrict__ k1) {
  __shared__ int s_warp[8];
  __shared__ int s_base;
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int nq = qc[p * qs];
  if (tid == 0) s_base = offsets[p];
  __syncthreads();
  for (int c0 = 0; c0 < nq; c0 += 256) {
    const int q = c0 + tid;
    const size_t o = static_cast<size_t>(p) * cap + q;
    const int g = q < nq ? good[o] : 0;
    const unsigned m = __ballot_sync(0xffffffffu, g);
    if (lane == 0) s_warp[wid] = __popc(m);
    __syncthreads();
    if (tid == 0) {
      int s = s_base;
      for (int w = 0; w < 8; ++w) { const int t = s_warp[w]; s_warp[w] = s; s += t; }
      s_base = s;
    }
    __syncthreads();
    if (g) {
      const int dst = s_warp[wid] + __popc(m & ((1u << lane) - 1u));
      const float* a = kp0 + (static_cast<size_t>(p) * s0 * cap + q) * 5;
      const float* c = kp1 + (static_cast<size_t>(p) * s1 * cap + i1[o]) * 5;
      k0[2 * dst] = a[0]; k0[2 * dst + 1] = a[1];
      k1[2 * dst] = c[0]; k1[2 * dst + 1] = c[1];
    }
    __syncthreads();
  }
}

// flag[p] = 1 when image 0 (counters c0, B0 images, index p * s0 + o0) or image 1 (c1, B1, p * s1 + o1) of pair p found more
// refined extrema or oriented keypoints than the capacity: its keypoints, and so the pair's matches, are then incomplete
__global__ void overflow_kernel(const int* __restrict__ c0, int B0, int s0, int o0, const int* __restrict__ c1, int B1, int s1,
                                int o1, int cap, int P, int* __restrict__ flag) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const int i0 = p * s0 + o0, i1 = p * s1 + o1;
  flag[p] = c0[i0] > cap || c0[B0 + i0] > cap || c1[i1] > cap || c1[B1 + i1] > cap;
}

// getGaussianKernel(ksize, sigma, CV_32F): exp in double, rounded to float, normalised in double, rounded again
Kernel1D gaussian_kernel(double sigma) {
  Kernel1D k{};
  const int ksize = static_cast<int>(std::lrint(sigma * 4 * 2 + 1)) | 1;
  k.r = ksize / 2;
  const double s2 = -0.5 / (sigma * sigma);
  double sum = 0;
  float cf[2 * kMaxR + 1];
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    cf[i] = static_cast<float>(std::exp(s2 * x * x));
    sum += cf[i];
  }
  sum = 1. / sum;
  for (int i = 0; i < ksize; ++i) k.c[i] = static_cast<float>(cf[i] * sum);
  return k;
}

}  // namespace

// the launch list's steps are grouped by stage: pyramid, extrema + refinement, orientation, selection, descriptors
struct SiftEngine : EngineCore {
  int B, H, W, nfeat, cap, cap2, root, nOct;
  int oh[kMaxOct], ow[kMaxOct];
  GraphExec graph;
  cudaStream_t own = nullptr;
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  unsigned char* img_u8 = nullptr;
  float* up = nullptr;
  float *gauss[kMaxOct], *dog[kMaxOct];
  int *counters = nullptr;   // [3][B]: extrema, oriented keypoints, selected
  float4* ext_f = nullptr; int4* ext_i = nullptr;
  float* kp = nullptr; int* kp_oct = nullptr;
  unsigned long long* keys = nullptr; int* sidx = nullptr; int* rank = nullptr;
  float* out_kp = nullptr; int* out_oct = nullptr; float* desc = nullptr;
  // match_pairs scratch
  int *m_i1 = nullptr, *m_i2 = nullptr, *pair_n = nullptr; float *m_d1 = nullptr, *m_d2 = nullptr; unsigned char* m_good = nullptr;

  void push(int stage, std::function<int(cudaStream_t)> f) { steps.push(std::move(f)).group = stage; }
  Pyr pyr() const {
    Pyr p{};
    p.n = nOct;
    for (int o = 0; o < nOct; ++o) { p.g[o] = gauss[o]; p.h[o] = oh[o]; p.w[o] = ow[o]; }
    return p;
  }

  int build() {
    nOct = static_cast<int>(std::lrint(std::log(static_cast<double>(std::min(2 * H, 2 * W))) / std::log(2.) - 2)) + 1;
    if (nOct < 1 || nOct > kMaxOct) return MFR_ERR_ARG;
    if (cudaStreamCreateWithFlags(&own, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ev_out, cudaEventDisableTiming) != cudaSuccess) return MFR_ERR_CUDA;
    cap2 = 1;
    while (cap2 < cap) cap2 <<= 1;
    oh[0] = 2 * H; ow[0] = 2 * W;
    for (int o = 1; o < nOct; ++o) { oh[o] = oh[o - 1] / 2; ow[o] = ow[o - 1] / 2; }
    img_u8 = mem.alloc<unsigned char>(static_cast<size_t>(B) * H * W);
    up = mem.alloc<float>(static_cast<size_t>(B) * oh[0] * ow[0], "upscaled");
    for (int o = 0; o < nOct; ++o) {
      const size_t plane = static_cast<size_t>(oh[o]) * ow[o];
      gauss[o] = mem.alloc<float>(static_cast<size_t>(B) * kLevels * plane, ("gauss_" + std::to_string(o)).c_str());
      dog[o] = mem.alloc<float>(static_cast<size_t>(B) * kDogs * plane, ("dog_" + std::to_string(o)).c_str());
    }
    counters = mem.alloc<int>(3 * B, "counters");
    const size_t bc = static_cast<size_t>(B) * cap;
    ext_f = mem.alloc<float4>(bc, "extrema_f"); ext_i = mem.alloc<int4>(bc, "extrema_i");
    kp = mem.alloc<float>(bc * 5, "kp_pre"); kp_oct = mem.alloc<int>(bc, "kp_pre_octave");
    keys = mem.alloc<unsigned long long>(static_cast<size_t>(B) * cap2); sidx = mem.alloc<int>(static_cast<size_t>(B) * cap2);
    rank = mem.alloc<int>(bc);
    out_kp = mem.alloc<float>(bc * 5, "keypoints"); out_oct = mem.alloc<int>(bc, "octaves"); desc = mem.alloc<float>(bc * 128, "descriptors");
    const int P = B / 2;
    if (P > 0) {
      const size_t pc = static_cast<size_t>(P) * cap;
      m_i1 = mem.alloc<int>(pc); m_i2 = mem.alloc<int>(pc); m_d1 = mem.alloc<float>(pc); m_d2 = mem.alloc<float>(pc);
      m_good = mem.alloc<unsigned char>(pc); pair_n = mem.alloc<int>(P);
    }
    if (rc != MFR_OK) return rc;

    // ---- pyramid (stage 0)
    const int nb = B, h0 = H, w0 = W;
    unsigned char* src = img_u8; float* upp = up;
    int* cnt = counters;
    push(0, [=](cudaStream_t st) { MFR_CUDA_CHECK(cudaMemsetAsync(cnt, 0, 3 * nb * sizeof(int), st)); return MFR_OK; });
    push(0, [=](cudaStream_t st) {
      for (int b = 0; b < nb; ++b) {   // the float path of cv2.resize(INTER_LINEAR) on the u8 image converted to float
        const int r = resize_linear(src + static_cast<size_t>(b) * h0 * w0, 1, w0, h0, w0, 1, upp + static_cast<size_t>(b) * 4 * h0 * w0,
                                    2 * w0, 2 * h0, 1, 1.f, 0, st);
        if (r != MFR_OK) return r;
      }
      return MFR_OK;
    });
    const float sig_diff = sqrtf(std::max(1.6f * 1.6f - 0.5f * 0.5f * 4, 0.01f));
    double sig[kLevels];
    sig[0] = 1.6;
    const double kk = std::pow(2., 1. / kLayers);
    for (int i = 1; i < kLevels; ++i) {
      const double prev = std::pow(kk, static_cast<double>(i - 1)) * 1.6, total = prev * kk;
      sig[i] = std::sqrt(total * total - prev * prev);
    }
    for (int o = 0; o < nOct; ++o) {
      const int h = oh[o], w = ow[o];
      const long long plane = static_cast<long long>(h) * w;
      float* G = gauss[o]; float* Dg = dog[o];
      const dim3 grid((w + kTile - 1) / kTile, (h + kTile - 1) / kTile, B), block(32, 8);
      if (o == 0) {
        const Kernel1D k = gaussian_kernel(sig_diff);
        push(0, [=](cudaStream_t st) {
          blur_kernel<<<grid, block, 0, st>>>(upp, plane, G, kLevels * plane, nullptr, 0, h, w, k);
          MFR_CUDA_CHECK(cudaGetLastError());
          return MFR_OK;
        });
      } else {
        const float* prev = gauss[o - 1] + static_cast<size_t>(kLayers) * oh[o - 1] * ow[o - 1];
        const long long pimg = static_cast<long long>(kLevels) * oh[o - 1] * ow[o - 1];
        const int sw = ow[o - 1];
        push(0, [=](cudaStream_t st) {
          downsample_kernel<<<dim3((w + 127) / 128, h, nb), 128, 0, st>>>(prev, pimg, sw, G, kLevels * plane, h, w);
          MFR_CUDA_CHECK(cudaGetLastError());
          return MFR_OK;
        });
      }
      for (int i = 1; i < kLevels; ++i) {
        const Kernel1D k = gaussian_kernel(sig[i]);
        push(0, [=](cudaStream_t st) {
          blur_kernel<<<grid, block, 0, st>>>(G + (i - 1) * plane, kLevels * plane, G + i * plane, kLevels * plane,
                                              Dg + (i - 1) * plane, kDogs * plane, h, w, k);
          MFR_CUDA_CHECK(cudaGetLastError());
          return MFR_OK;
        });
      }
    }
    // ---- extrema + refinement (stage 1)
    const int cp = cap;
    float4* ef = ext_f; int4* ei = ext_i;
    for (int o = 0; o < nOct; ++o) {
      const int h = oh[o], w = ow[o];
      if (h <= 2 * kBorder || w <= 2 * kBorder) continue;
      const float* Dg = dog[o];
      const dim3 grid((w + 31) / 32, (h + 7) / 8, B * kLayers), block(32, 8);
      push(1, [=](cudaStream_t st) {
        extrema_kernel<<<grid, block, 0, st>>>(Dg, h, w, o, cp, cnt, ef, ei);
        MFR_CUDA_CHECK(cudaGetLastError());
        return MFR_OK;
      });
    }
    // ---- orientation (stage 2)
    const Pyr py = pyr();
    float* kpp = kp; int* kpo = kp_oct;
    push(2, [=](cudaStream_t st) {
      orientation_kernel<<<dim3(std::min((cp + kOriWarps - 1) / kOriWarps, 512), nb), kOriWarps * 32, 0, st>>>(
          py, cnt, ef, ei, cp, cnt + nb, kpp, kpo);
      MFR_CUDA_CHECK(cudaGetLastError());
      return MFR_OK;
    });
    // ---- selection (stage 3)
    const int c2 = cap2, nf = nfeat;
    unsigned long long* kys = keys; int* si = sidx; int* rk = rank; float* okp = out_kp; int* oo = out_oct;
    push(3, [=](cudaStream_t st) {
      select_kernel<<<nb, kSelThreads, 0, st>>>(cnt + nb, kpp, kpo, cp, c2, kys, si, rk, nf, cnt + 2 * nb, okp, oo);
      MFR_CUDA_CHECK(cudaGetLastError());
      return MFR_OK;
    });
    // ---- descriptors (stage 4)
    const int rt = root; float* ds = desc;
    push(4, [=](cudaStream_t st) {
      descriptor_kernel<<<dim3(std::min(cp, 1024), nb), kDescThreads, 0, st>>>(py, cnt + 2 * nb, okp, oo, cp, rt, ds);
      MFR_CUDA_CHECK(cudaGetLastError());
      return MFR_OK;
    });
    return rc;
  }

  // The launch list runs on the engine's own stream, ordered after / before the caller's stream by events: a graph
  // cannot be captured on the legacy default stream a caller may pass.
  int detect(const unsigned char* imgs, cudaStream_t st) {
    if (!imgs) return MFR_ERR_ARG;
    MFR_CUDA_CHECK(cudaEventRecord(ev_in, st));
    MFR_CUDA_CHECK(cudaStreamWaitEvent(own, ev_in, 0));
    MFR_CUDA_CHECK(cudaMemcpyAsync(img_u8, imgs, static_cast<size_t>(B) * H * W, cudaMemcpyDeviceToDevice, own));
    const int r = graph.launch(steps, own, use_graph, "sift");
    if (r != MFR_OK) return r;
    MFR_CUDA_CHECK(cudaEventRecord(ev_out, own));
    MFR_CUDA_CHECK(cudaStreamWaitEvent(st, ev_out, 0));
    return MFR_OK;
  }
  // eager run with an event pair around each stage: ms[5] = pyramid, extrema + refinement, orientation, selection, descriptors
  int profile(const unsigned char* imgs, float* ms, cudaStream_t st) {
    if (!imgs || !ms) return MFR_ERR_ARG;
    MFR_CUDA_CHECK(cudaMemcpyAsync(img_u8, imgs, static_cast<size_t>(B) * H * W, cudaMemcpyDeviceToDevice, st));
    std::vector<float> t;
    const int r = timed_run(steps, st, t);
    if (r == MFR_OK) std::copy(t.begin(), t.end(), ms);
    return r;
  }

  int match_pairs(float ratio, float* k0, float* k1, int* offsets, cudaStream_t st) {
    const int P = B / 2;
    if (P < 1 || (B & 1) || !k0 || !k1 || !offsets) return MFR_ERR_ARG;
    int* cnt = counters + 2 * B;
    int r = knn2_l2_pairs(desc, cnt, P, cap, 128, m_i1, m_d1, m_i2, m_d2, st);
    if (r != MFR_OK) return r;
    ratio_count_kernel<<<P, 256, 0, st>>>(cnt, 2, cnt + 1, 2, m_d1, m_d2, cap, ratio, m_good, pair_n);
    pair_offsets_kernel<<<1, 32, 0, st>>>(pair_n, P, offsets);
    compact_matches_kernel<<<P, 256, 0, st>>>(cnt, 2, m_good, m_i1, out_kp, 2, out_kp + static_cast<size_t>(cap) * 5, 2, cap,
                                              offsets, k0, k1);
    MFR_CUDA_CHECK(cudaGetLastError());
    return MFR_OK;
  }

  ~SiftEngine() {
    if (own) cudaStreamDestroy(own);
    if (ev_in) cudaEventDestroy(ev_in);
    if (ev_out) cudaEventDestroy(ev_out);
  }
};

int sift_create(int B, int H, int W, int nfeatures, int max_candidates, int root_sift, SiftEngine** out) {
  if (!out || B < 1 || H < 1 || W < 1 || nfeatures < 0 || max_candidates < 1 || max_candidates > (1 << 22)) return MFR_ERR_ARG;
  auto* e = new SiftEngine();
  e->B = B; e->H = H; e->W = W; e->nfeat = nfeatures; e->cap = max_candidates; e->root = root_sift != 0;
  const int rc = e->build();
  if (rc != MFR_OK) { delete e; return rc; }
  *out = e;
  return MFR_OK;
}
void sift_destroy(SiftEngine* e) { delete e; }
EngineCore& engine_core(SiftEngine* e) { return *e; }
int sift_detect(SiftEngine* e, const unsigned char* imgs, cudaStream_t st) { return e->detect(imgs, st); }
void sift_outputs(SiftEngine* e, mfr_sift_outputs* o) {
  o->counts = e->counters + 2 * e->B; o->raw_counts = e->counters + e->B; o->extrema_counts = e->counters;
  o->keypoints = e->out_kp; o->octaves = e->out_oct; o->descriptors = e->desc; o->capacity = e->cap;
}
int sift_match_pairs(SiftEngine* e, float ratio, float* kpts0, float* kpts1, int* offsets, cudaStream_t st) {
  return e->match_pairs(ratio, kpts0, kpts1, offsets, st);
}
int sift_profile(SiftEngine* e, const unsigned char* imgs, float* ms, cudaStream_t st) { return e->profile(imgs, ms, st); }

// P pairs as a pair engine: detection of the 2P pair-interleaved images (image 2p = img0[p], 2p + 1 = img1[p]), 2-NN,
// ratio test, offsets and the ordered compaction, in one launch list replayed as one CUDA graph, with no host
// synchronisation. The kernels and their inputs are those of SiftEngine::detect + match_pairs, so the outputs are the
// same bits. The shared-map path detects the map once (its own B = 1 engine, eagerly) and the P queries in a B = P
// engine; per-image detection does not depend on the batch, so it gives the bits of the paired path with the map
// repeated.
struct SiftPairs : EngineCore {
  int P = 0, cap = 0;
  float ratio = 0.8f;
  SiftEngine *pair = nullptr, *query = nullptr, *map = nullptr;
  float *k0 = nullptr, *k1 = nullptr;
  int *offsets = nullptr, *overflow = nullptr;
  bool map_set = false;
  LaunchList shared_steps;
  GraphExec graph, shared_graph;

  // the matching half: knn + ratio test + offsets + compaction + overflow flags, appended to a detection list
  void push_match(LaunchList& list, const float* d0, const int* qc, int qs, const float* kp0, int s0, const float* d1,
                  const int* tc, int ts, const float* kp1, int s1, bool shared, const int* c0, int B0, int cs0, int co0,
                  const int* c1, int B1, int cs1, int co1) {
    const int np = P, cp = cap;
    const float rt = ratio;
    int *i1 = pair->m_i1, *i2 = pair->m_i2, *pn = pair->pair_n, *off = offsets, *ov = overflow;
    float *dd1 = pair->m_d1, *dd2 = pair->m_d2, *o0 = k0, *o1 = k1;
    unsigned char* good = pair->m_good;
    list.push([=](cudaStream_t st) {
      return shared ? knn2_l2_shared(d0, qc, d1, tc, np, cp, 128, i1, dd1, i2, dd2, st)
                    : knn2_l2_pairs(d0, qc, np, cp, 128, i1, dd1, i2, dd2, st);
    }, "knn2");
    list.push([=](cudaStream_t st) {
      ratio_count_kernel<<<np, 256, 0, st>>>(qc, qs, tc, ts, dd1, dd2, cp, rt, good, pn);
      pair_offsets_kernel<<<1, 32, 0, st>>>(pn, np, off);
      compact_matches_kernel<<<np, 256, 0, st>>>(qc, qs, good, i1, kp0, s0, kp1, s1, cp, off, o0, o1);
      overflow_kernel<<<(np + 127) / 128, 128, 0, st>>>(c0, B0, cs0, co0, c1, B1, cs1, co1, cp, np, ov);
      MFR_CUDA_CHECK(cudaGetLastError());
      return MFR_OK;
    }, "ratio_compact", 4);
  }

  int build(int H, int W, int nfeat, int root) {
    int r = sift_create(2 * P, H, W, nfeat, cap, root, &pair);
    if (r == MFR_OK) r = sift_create(P, H, W, nfeat, cap, root, &query);
    if (r == MFR_OK) r = sift_create(1, H, W, nfeat, cap, root, &map);
    if (r != MFR_OK) return r;
    const size_t pc = static_cast<size_t>(P) * cap;
    k0 = mem.alloc<float>(pc * 2, "kpts0"); k1 = mem.alloc<float>(pc * 2, "kpts1");
    offsets = mem.alloc<int>(P + 1, "offsets"); overflow = mem.alloc<int>(P, "overflow");
    if (rc != MFR_OK) return rc;
    // paired: image 0 of pair p is image 2p of the pair engine, image 1 is 2p + 1
    steps.append(pair->steps, 0, pair->steps.size());
    const int B2 = 2 * P;
    const int* pc_sel = pair->counters + 2 * B2;
    push_match(steps, pair->desc, pc_sel, 2, pair->out_kp, 2, pair->desc + static_cast<size_t>(cap) * 128, pc_sel + 1, 2,
               pair->out_kp + static_cast<size_t>(cap) * 5, 2, false, pair->counters, B2, 2, 0, pair->counters, B2, 2, 1);
    // shared: image 0 of every pair is the map image (stride 0), image 1 of pair p is query image p
    shared_steps.append(query->steps, 0, query->steps.size());
    const int* mc_sel = map->counters + 2;
    const int* qc_sel = query->counters + 2 * P;
    push_match(shared_steps, map->desc, mc_sel, 0, map->out_kp, 0, query->desc, qc_sel, 1, query->out_kp, 1, true,
               map->counters, 1, 0, 0, query->counters, P, 1, 0);
    return rc;
  }

  // img0 / img1: device uint8 [P][H][W], staged into the pair-interleaved input (the graph does not depend on their
  // addresses)
  int forward_pairs(const unsigned char* img0, const unsigned char* img1, cudaStream_t st) {
    if (!img0 || !img1) return MFR_ERR_ARG;
    const size_t hw = static_cast<size_t>(pair->H) * pair->W;
    MFR_CUDA_CHECK(cudaMemcpy2DAsync(pair->img_u8, 2 * hw, img0, hw, hw, P, cudaMemcpyDeviceToDevice, st));
    MFR_CUDA_CHECK(cudaMemcpy2DAsync(pair->img_u8 + hw, 2 * hw, img1, hw, hw, P, cudaMemcpyDeviceToDevice, st));
    return graph.launch(steps, st, use_graph, "sift_pairs");
  }
  int set_map(const unsigned char* img0, cudaStream_t st) {
    if (!img0) return MFR_ERR_ARG;
    map_set = false;
    MFR_CUDA_CHECK(cudaMemcpyAsync(map->img_u8, img0, static_cast<size_t>(map->H) * map->W, cudaMemcpyDeviceToDevice, st));
    const int r = map->steps.run(st);
    if (r != MFR_OK) return r;
    map_set = true;
    return MFR_OK;
  }
  int forward_shared(const unsigned char* img1, cudaStream_t st) {
    if (!img1 || !map_set) return MFR_ERR_ARG;
    MFR_CUDA_CHECK(cudaMemcpyAsync(query->img_u8, img1, static_cast<size_t>(P) * query->H * query->W, cudaMemcpyDeviceToDevice, st));
    return shared_graph.launch(shared_steps, st, use_graph, "sift_pairs_shared");
  }

  ~SiftPairs() {
    delete pair; delete query; delete map;
  }
};

int sift_pairs_create(int P, int H, int W, int nfeatures, int max_candidates, int root_sift, float ratio, SiftPairs** out) {
  if (!out || P < 1 || !(ratio > 0.f)) return MFR_ERR_ARG;
  auto* e = new SiftPairs();
  e->P = P; e->cap = max_candidates; e->ratio = ratio;
  const int rc = e->build(H, W, nfeatures, root_sift);
  if (rc != MFR_OK) { delete e; return rc; }
  *out = e;
  return MFR_OK;
}
void sift_pairs_destroy(SiftPairs* e) { delete e; }
EngineCore& engine_core(SiftPairs* e) { return *e; }
int sift_forward_pairs(SiftPairs* e, const unsigned char* img0, const unsigned char* img1, cudaStream_t st) {
  return e->forward_pairs(img0, img1, st);
}
int sift_pairs_set_map(SiftPairs* e, const unsigned char* img0, cudaStream_t st) { return e->set_map(img0, st); }
int sift_forward_shared(SiftPairs* e, const unsigned char* img1, cudaStream_t st) { return e->forward_shared(img1, st); }
void sift_pair_outputs(SiftPairs* e, mfr_sift_pair_outputs* o) {
  o->kpts0 = e->k0; o->kpts1 = e->k1; o->offsets = e->offsets; o->overflow = e->overflow;
  o->capacity = e->P * e->cap; o->max_pts_per_pair = e->cap;
}


}  // namespace mfr
