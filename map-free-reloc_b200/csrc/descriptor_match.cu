// Exact brute-force 2-nearest-neighbour search between two descriptor sets (L2), the matching half
// of the reference's SIFT plugin (lib/models/matching/feature_matching.py:87-99,
// etc/feature_matching_baselines/matchers.py:158-175): knnMatch(k=2) + Lowe ratio test. The
// reference uses an approximate, non-deterministic FLANN kd-tree; this kernel is the exact search
// (= cv2.BFMatcher(NORM_L2).knnMatch), so integer match indices are reproducible bit for bit.
#include "descriptor_match.cuh"

#include <algorithm>

namespace mfr {

namespace {

struct Best2 {
  float d1, d2;
  int i1, i2;
};

__device__ __forceinline__ void push(Best2& b, float d, int j) {
  // lexicographic (distance, index): the lowest index wins ties, like a linear scan
  if (d < b.d1 || (d == b.d1 && j < b.i1)) {
    b.d2 = b.d1; b.i2 = b.i1; b.d1 = d; b.i1 = j;
  } else if (d < b.d2 || (d == b.d2 && j < b.i2)) {
    b.d2 = d; b.i2 = j;
  }
}

// one block (128 threads) per query descriptor (grid-stride over queries); dim <= 256 and a multiple of 4.
// blockIdx.y = pair p: its queries / train rows / outputs start p * q_stride / t_stride / o_stride rows in, and
// with `qc` / `tc` non-null the row counts are qc[p * qc_stride] (queries) / tc[p * tc_stride] (train), read on the device.
__global__ void __launch_bounds__(128, 8) knn2_kernel(const float* __restrict__ q, int nq,
                                                   const float* __restrict__ t, int nt, int dim,
                                                   int* __restrict__ idx1, float* __restrict__ dist1,
                                                   int* __restrict__ idx2, float* __restrict__ dist2,
                                                   long long q_stride, long long t_stride, long long o_stride,
                                                   const int* __restrict__ qc, int qc_stride,
                                                   const int* __restrict__ tc, int tc_stride) {
  __shared__ __align__(16) float sq[256];
  __shared__ Best2 sb[4];
  const int p = blockIdx.y;
  if (qc) nq = qc[p * qc_stride];
  if (tc) nt = tc[p * tc_stride];
  q += p * q_stride * dim; t += p * t_stride * dim;
  idx1 += p * o_stride; dist1 += p * o_stride; idx2 += p * o_stride; dist2 += p * o_stride;
  for (int qi = blockIdx.x; qi < nq; qi += gridDim.x) {
  __syncthreads();
  for (int k = threadIdx.x; k < dim; k += blockDim.x) sq[k] = q[static_cast<size_t>(qi) * dim + k];
  __syncthreads();
  Best2 b{3.0e38f, 3.0e38f, 0x7fffffff, 0x7fffffff};
  const int d4 = dim >> 2;
  for (int j = threadIdx.x; j < nt; j += blockDim.x) {
    const float4* tr = reinterpret_cast<const float4*>(t + static_cast<size_t>(j) * dim);
    float acc = 0.f;
    for (int k = 0; k < d4; ++k) {
      const float4 a = reinterpret_cast<const float4*>(sq)[k];
      const float4 c = __ldg(tr + k);
      const float dx = a.x - c.x, dy = a.y - c.y, dz = a.z - c.z, dw = a.w - c.w;
      acc = fmaf(dx, dx, acc); acc = fmaf(dy, dy, acc); acc = fmaf(dz, dz, acc); acc = fmaf(dw, dw, acc);
    }
    push(b, acc, j);
  }
  // warp merge, then block merge
  for (int o = 16; o > 0; o >>= 1) {
    Best2 ob;
    ob.d1 = __shfl_xor_sync(0xffffffffu, b.d1, o); ob.i1 = __shfl_xor_sync(0xffffffffu, b.i1, o);
    ob.d2 = __shfl_xor_sync(0xffffffffu, b.d2, o); ob.i2 = __shfl_xor_sync(0xffffffffu, b.i2, o);
    if (ob.i1 != 0x7fffffff) push(b, ob.d1, ob.i1);
    if (ob.i2 != 0x7fffffff) push(b, ob.d2, ob.i2);
  }
  if ((threadIdx.x & 31) == 0) sb[threadIdx.x >> 5] = b;
  __syncthreads();
  if (threadIdx.x == 0) {
    Best2 r = sb[0];
    for (int w = 1; w < 4; ++w) {
      if (sb[w].i1 != 0x7fffffff) push(r, sb[w].d1, sb[w].i1);
      if (sb[w].i2 != 0x7fffffff) push(r, sb[w].d2, sb[w].i2);
    }
    idx1[qi] = r.i1 == 0x7fffffff ? -1 : r.i1;
    idx2[qi] = r.i2 == 0x7fffffff ? -1 : r.i2;
    dist1[qi] = sqrtf(r.d1);
    dist2[qi] = sqrtf(r.d2);
  }
  }
}

}  // namespace

int knn2_l2(const float* q, int nq, const float* t, int nt, int dim, int* idx1, float* dist1, int* idx2,
            float* dist2, cudaStream_t st) {
  if (nq <= 0) return MFR_OK;
  if (dim > 256 || (dim & 3) || nt < 0) return MFR_ERR_ARG;
  knn2_kernel<<<nq, 128, 0, st>>>(q, nq, t, nt, dim, idx1, dist1, idx2, dist2, 0, 0, 0, nullptr, 0, nullptr, 0);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int knn2_l2_pairs(const float* desc, const int* counts, int P, int cap, int dim, int* idx1, float* dist1, int* idx2,
                  float* dist2, cudaStream_t st) {
  if (P <= 0 || cap <= 0) return MFR_OK;
  if (dim > 256 || (dim & 3)) return MFR_ERR_ARG;
  const dim3 grid(std::min(cap, 1024), P);
  knn2_kernel<<<grid, 128, 0, st>>>(desc, cap, desc + static_cast<size_t>(cap) * dim, cap, dim, idx1, dist1, idx2, dist2,
                                    2LL * cap, 2LL * cap, cap, counts, 2, counts + 1, 2);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int knn2_l2_shared(const float* q, const int* q_count, const float* t, const int* t_counts, int P, int cap, int dim,
                   int* idx1, float* dist1, int* idx2, float* dist2, cudaStream_t st) {
  if (P <= 0 || cap <= 0) return MFR_OK;
  if (dim > 256 || (dim & 3)) return MFR_ERR_ARG;
  const dim3 grid(std::min(cap, 1024), P);
  knn2_kernel<<<grid, 128, 0, st>>>(q, cap, t, cap, dim, idx1, dist1, idx2, dist2, 0, cap, cap, q_count, 0, t_counts, 1);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

}  // namespace mfr
