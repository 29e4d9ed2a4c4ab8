// Pose back end on the GPU: batched-hypothesis RANSAC for the essential matrix (5-point) and for
// PnP (P3P), local optimisation, cheirality, depth lift and the scale consensus.
// Replaces the OpenCV calls of the reference's lib/models/matching/pose_solver.py:
//   EssentialMatrixSolver.estimate_pose        :29-61   -> emat_ransac
//   EssentialMatrixMetricSolver.estimate_pose  :125-172 -> scale_from_depth
//   PnPSolver.estimate_pose                    :184-235 -> pnp_ransac
// Hypothesis kernels: every lane of a warp draws its own minimal sample and solves it in fp64
// registers/local memory (fixed work bound, no complex arithmetic); the warp then scores its 32
// hypotheses one after the other with all lanes striding over the correspondences held in shared
// memory, inlier counts via __ballot_sync/__popc. Thousands of hypotheses per pair, many pairs per
// launch (grid.y = pair).
#include "geometry.cuh"

#include <algorithm>
#include <cstddef>
#include <cstring>

#include "geometry_solvers.cuh"

namespace mfr {

namespace {

using namespace geo;

constexpr int kHypPerBlock = 128;  // 4 warps x 32 lanes

// Scoring rule of the E-mat RANSAC, a compile-time policy of its three kernels:
//   kMsac   sum min(d^2, thr^2) ranks the hypotheses; LO = LM on a Tukey M-estimator + noise-adaptive tightening (+ the
//           truncated least-squares refit), as lo_enabled asks (mfr_emat_ransac)
//   kMagsac sum rho, the MAGSAC++ loss with sigma_max = thr (geometry_solvers.cuh), ranks the hypotheses; LO and the
//           final polish are sigma-consensus++, i.e. IRLS / LM on sum rho (mfr_emat_magsac)
enum class Scoring { kMsac, kMagsac };

struct HypResult {   // best hypothesis of one block
  double cost;       // MSAC cost or sum of MAGSAC++ rho (emat), -inlier count (pnp): lower is better
  int count;
  int valid;
  double model[12];  // E[9] or R[9] t[3]
};
// the layout tests read through pose_solver_debug_tensor("hyp_results") as a numpy structured dtype
static_assert(sizeof(HypResult) == 112 && offsetof(HypResult, cost) == 0 && offsetof(HypResult, count) == 8 &&
                  offsetof(HypResult, valid) == 12 && offsetof(HypResult, model) == 16,
              "HypResult layout is part of the debug interface");

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long& s) {
  s += 0x9E3779B97F4A7C15ull;
  unsigned long long z = s;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

template <int K>
__device__ __forceinline__ void sample_distinct(unsigned long long& st, int n, int* idx) {
  for (int k = 0; k < K; ++k) {
    int v = 0;
    for (int tries = 0; tries < 64; ++tries) {
      v = static_cast<int>(splitmix64(st) % static_cast<unsigned long long>(n));
      bool dup = false;
      for (int j = 0; j < k; ++j) dup |= (idx[j] == v);
      if (!dup) break;
    }
    idx[k] = v;
  }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum of K doubles per thread (blockDim.x <= 512); result valid in thread 0
template <int K>
__device__ __forceinline__ void block_sum_256(double (&v)[K], double* sh /*[(blockDim.x / 32) * K]*/) {
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = warp_sum_d(v[k]);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
    for (int k = 0; k < K; ++k) sh[w * K + k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int k = 0; k < K; ++k) {
      double s = 0.0;
      for (int ww = 0; ww < static_cast<int>(blockDim.x >> 5); ++ww) s += sh[ww * K + k];
      v[k] = s;
    }
  __syncthreads();
}

// float32 normalisation exactly as numpy does it on float32 arrays (pose_solver.py:39-40)
__device__ __forceinline__ float4 normalise_pt(const float* k0, const float* k1, int i, const float* K0,
                                               const float* K1) {
  float4 p;
  p.x = __fdiv_rn(__fsub_rn(k0[2 * i], K0[2]), K0[0]);
  p.y = __fdiv_rn(__fsub_rn(k0[2 * i + 1], K0[5]), K0[4]);
  p.z = __fdiv_rn(__fsub_rn(k1[2 * i], K1[2]), K1[0]);
  p.w = __fdiv_rn(__fsub_rn(k1[2 * i + 1], K1[5]), K1[4]);
  return p;
}
// pose_solver.py:43 in float32
__device__ __forceinline__ float emat_threshold(float pix_thr, const float* K0, const float* K1) {
  const float m = __fmul_rn(__fadd_rn(__fadd_rn(K0[0], K1[4]), __fadd_rn(K0[4], K1[0])), 0.25f);
  return __fdiv_rn(pix_thr, m);
}

__device__ __forceinline__ float sampson_sq_f(const float* E, float4 p) {
  const float a0 = fmaf(E[0], p.x, fmaf(E[1], p.y, E[2]));
  const float a1 = fmaf(E[3], p.x, fmaf(E[4], p.y, E[5]));
  const float a2 = fmaf(E[6], p.x, fmaf(E[7], p.y, E[8]));
  const float b0 = fmaf(E[0], p.z, fmaf(E[3], p.w, E[6]));
  const float b1 = fmaf(E[1], p.z, fmaf(E[4], p.w, E[7]));
  const float num = fmaf(p.z, a0, fmaf(p.w, a1, a2));
  const float den = fmaf(a0, a0, fmaf(a1, a1, fmaf(b0, b0, b1 * b1)));
  return __fdividef(num * num, den);
}

// ================================================================================================
// essential matrix: hypothesis generation + scoring
// ================================================================================================
// normalised correspondences of every pair, once, for the hypothesis kernel: pts[pair][i] = (K0^-1 x0, K1^-1 x1)
__global__ void __launch_bounds__(256) emat_normalise_kernel(const float* __restrict__ kpts0, const float* __restrict__ kpts1,
                                                             const int* __restrict__ offsets, const float* __restrict__ K0s,
                                                             const float* __restrict__ K1s, int max_pts,
                                                             float4* __restrict__ pts) {
  const int pair = blockIdx.y;
  const int n0 = offsets[pair];
  const int N = min(offsets[pair + 1] - n0, max_pts);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  pts[static_cast<size_t>(pair) * max_pts + i] = normalise_pt(kpts0 + 2 * static_cast<size_t>(n0), kpts1 + 2 * static_cast<size_t>(n0), i,
                                                              K0s + 9 * pair, K1s + 9 * pair);
}

// The hypothesis kernel is the long one of the back end (a 5-point solve is ~1.8 ms of dependent fp64 work) and runs on
// the solver stream under the next batch's matcher, whose persistent GEMM CTAs hold all but 2 KB of an SM's shared
// memory and all but ~21 K of its registers. It therefore keeps out of shared memory (the points come through L1 / L2,
// 32 bytes of block-reduction scratch) and under 160 registers, so that one of its blocks fits NEXT to a GEMM CTA
// instead of making that CTA (and, with static tile assignment, the whole GEMM kernel) wait for it.
template <Scoring kScore>
__global__ void __maxnreg__(160) emat_hyp_kernel(   // launched with <= kHypPerBlock threads
    const float4* __restrict__ pts_all, const int* __restrict__ offsets,
    const float* __restrict__ K0s, const float* __restrict__ K1s, float pix_thr, int num_hyp,
    unsigned long long seed, int max_pts, HypResult* __restrict__ results, const int* __restrict__ active) {
  __shared__ double s_cost[kHypPerBlock / 32];
  const int pair = blockIdx.y;
  if (active && !active[pair]) return;
  const int n0 = offsets[pair];
  const int N = min(offsets[pair + 1] - n0, max_pts);
  HypResult* out = results + static_cast<size_t>(pair) * gridDim.x + blockIdx.x;
  if (N < 5) {
    if (threadIdx.x == 0) { out->valid = 0; out->cost = 1e300; out->count = 0; }
    return;
  }
  const float* K0 = K0s + 9 * pair;
  const float* K1 = K1s + 9 * pair;
  const float4* s_pts = pts_all + static_cast<size_t>(pair) * max_pts;
  const float thr = emat_threshold(pix_thr, K0, K1);
  const float thr2 = thr * thr;
  const float inv2s2 = 0.5f / thr2;   // MAGSAC++: x = d^2 / (2 sigma_max^2); the scores are sums of rho / (C 2^1.5 thr)

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.x * blockDim.x + threadIdx.x;   // 32..128 hypotheses per block (host picks, to fill the SMs)
  double Ec[10][9];
  int ncand = 0;
  if (h < num_hyp) {
    unsigned long long st = seed ^ (0xD1B54A32D192ED03ull * (static_cast<unsigned long long>(pair) + 1)) ^
                            (0x9E3779B97F4A7C15ull * (static_cast<unsigned long long>(h) + 1));
    int idx[5];
    sample_distinct<5>(st, N, idx);
    double x0[5][2], x1[5][2];
    for (int k = 0; k < 5; ++k) {
      const float4 p = __ldg(s_pts + idx[k]);
      x0[k][0] = p.x; x0[k][1] = p.y; x1[k][0] = p.z; x1[k][1] = p.w;
    }
    ncand = five_point(x0, x1, Ec);
  }
  // ---- scoring: the warp walks over its 32 hypotheses
  float best_cost = 3.0e38f;
  int best_cnt = 0, best_src = -1, best_c = 0;
  for (int src = 0; src < 32; ++src) {
    const int cnt = __shfl_sync(0xffffffffu, ncand, src);
    for (int c = 0; c < cnt; ++c) {
      float E[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) E[k] = __shfl_sync(0xffffffffu, static_cast<float>(Ec[c][k]), src);
      float cost = 0.f;
      int inl = 0;
      bool dead = false;
      for (int i0 = 0; i0 < N; i0 += 128) {
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = i0 + u * 32 + lane;
          float d2 = thr2;
          bool ok = false;
          if (i < N) {
            d2 = sampson_sq_f(E, __ldg(s_pts + i));
            ok = d2 < thr2;
            if constexpr (kScore == Scoring::kMsac)
              cost += fminf(d2, thr2);
            else
              cost += magsac_rho_unit_f(d2 * inv2s2);
          }
          inl += __popc(__ballot_sync(0xffffffffu, ok));
        }
        // the cost (MSAC or MAGSAC++: rho >= 0) only grows: give up on this model once it cannot beat the best so far
        const float partial = warp_sum_f(cost);
        if (partial >= best_cost) { dead = true; break; }
      }
      if (dead) continue;
      const float total = warp_sum_f(cost);
      if (total < best_cost) {
        best_cost = total;
        best_cnt = inl;
        best_src = src;
        best_c = c;
      }
    }
  }
  // block winner = the warp with the lowest cost (first one on ties); that warp writes the record itself
  if constexpr (kScore == Scoring::kMagsac) best_cost *= static_cast<float>(kMagsacC2) * thr;   // sum rho
  if (lane == 0) s_cost[warp] = best_src >= 0 ? static_cast<double>(best_cost) : 1e300;
  __syncthreads();
  int bw = 0;
  for (int w = 1; w < static_cast<int>(blockDim.x) / 32; ++w)
    if (s_cost[w] < s_cost[bw]) bw = w;
  if (warp != bw) return;
  if (lane == 0) {
    out->valid = best_src >= 0 ? 1 : 0;
    out->cost = best_src >= 0 ? static_cast<double>(best_cost) : 1e300;
    out->count = best_cnt;
  }
  if (best_src >= 0 && lane == best_src)
    for (int k = 0; k < 9; ++k) out->model[k] = Ec[best_c][k];
}

// ------------------------------------------------------------------------------------------------
// Sampson residual and its Jacobian w.r.t. (d_omega[3], d_tau[2]) for E = [t]x R
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tangent_basis(const double* t, double* b1, double* b2) {
  double a[3] = {0, 0, 0};
  const double ax = fabs(t[0]), ay = fabs(t[1]), az = fabs(t[2]);
  if (ax <= ay && ax <= az) a[0] = 1.0; else if (ay <= az) a[1] = 1.0; else a[2] = 1.0;
  cross3(t, a, b1);
  const double n = norm3(b1);
  for (int k = 0; k < 3; ++k) b1[k] /= n;
  cross3(t, b1, b2);
}

__device__ __forceinline__ double sampson_res_jac(const double* R, const double* t, const double* b1,
                                                  const double* b2, float4 p, double* J) {
  const double x0[3] = {p.x, p.y, 1.0}, x1[3] = {p.z, p.w, 1.0};
  double y[3], w[3], a[3], b[3], tmp[3];
  mat3_vec(R, x0, y);   // y = R x0
  cross3(t, y, a);      // a = E x0 = t x (R x0)
  cross3(t, x1, w);     // w = t x x1 ; E^T x1 = -R^T w
  // b = E^T x1 = R^T [t]x^T x1 = -R^T (t x x1)
  for (int i = 0; i < 3; ++i) b[i] = -(R[i] * w[0] + R[3 + i] * w[1] + R[6 + i] * w[2]);
  const double n = dot3(x1, a);
  const double s = a[0] * a[0] + a[1] * a[1] + b[0] * b[0] + b[1] * b[1];
  const double is = 1.0 / sqrt(s);
  const double r = n * is;
  const double c2 = -0.5 * n * is * is * is;
  for (int k = 0; k < 5; ++k) {
    double da[3], db[3];
    if (k < 3) {
      double ek[3] = {0, 0, 0};
      ek[k] = 1.0;
      cross3(ek, y, tmp);
      cross3(t, tmp, da);                 // da = t x (e_k x y)
      cross3(ek, w, tmp);                 // db = R^T (e_k x w)
      for (int i = 0; i < 3; ++i) db[i] = R[i] * tmp[0] + R[3 + i] * tmp[1] + R[6 + i] * tmp[2];
    } else {
      const double* bj = (k == 3) ? b1 : b2;
      cross3(bj, y, da);                  // da = b_j x y
      cross3(bj, x1, tmp);                // db = -R^T (b_j x x1)
      for (int i = 0; i < 3; ++i) db[i] = -(R[i] * tmp[0] + R[3 + i] * tmp[1] + R[6 + i] * tmp[2]);
    }
    const double dn = dot3(x1, da);
    const double ds = 2.0 * (a[0] * da[0] + a[1] * da[1] + b[0] * db[0] + b[1] * db[1]);
    J[k] = dn * is + c2 * ds;
  }
  return r;
}

// cheirality of one correspondence for a candidate (R, t): both depths positive
__device__ __forceinline__ bool cheirality_ok(const double* R, const double* t, float4 p) {
  const double d0[3] = {p.x, p.y, 1.0}, d1[3] = {p.z, p.w, 1.0};
  double a[3];
  mat3_vec(R, d0, a);
  const double aa = dot3(a, a), bb = dot3(d1, d1), ab = dot3(a, d1), at = dot3(a, t), bt = dot3(d1, t);
  const double det = aa * bb - ab * ab;
  if (!(fabs(det) > 1e-300)) return false;
  const double l0 = (-at * bb + ab * bt) / det;
  const double l1 = (aa * bt - ab * at) / det;
  return l0 > 0.0 && l1 > 0.0 && l0 < 1e9 && l1 < 1e9;
}

// solve (H + lambda diag(H)) d = -g for an n x n SPD system stored full (row-major, n <= 6)
__device__ inline bool solve_damped(const double* H, const double* g, double lambda, int n, double* d) {
  double A[6][7];
  for (int i = 0; i < n; ++i) {
    for (int j = 0; j < n; ++j) A[i][j] = H[i * n + j];
    A[i][i] += lambda * (H[i * n + i] + 1e-12);
    A[i][n] = -g[i];
  }
  for (int k = 0; k < n; ++k) {
    int pr = k;
    for (int i = k + 1; i < n; ++i)
      if (fabs(A[i][k]) > fabs(A[pr][k])) pr = i;
    if (fabs(A[pr][k]) < 1e-300) return false;
    if (pr != k)
      for (int j = 0; j <= n; ++j) { const double tt = A[k][j]; A[k][j] = A[pr][j]; A[pr][j] = tt; }
    for (int i = k + 1; i < n; ++i) {
      const double f = A[i][k] / A[k][k];
      for (int j = k; j <= n; ++j) A[i][j] -= f * A[k][j];
    }
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = A[i][n];
    for (int j = i + 1; j < n; ++j) s -= A[i][j] * d[j];
    d[i] = s / A[i][i];
  }
  return true;
}

// ================================================================================================
// essential matrix: top-K block winners -> local optimisation -> best final model, cheirality, mask
// ================================================================================================
constexpr int kLoRounds = 6, kLoInner = 5, kLoTopK = 4, kTightRounds = 3;

struct EmatShared {
  double R[9], t[3], E[9], prevR[9], prevt[3], H[25], g[5];
  double bestR[9], bestt[3], best_cost;
  double c_R1[9], c_R2[9], c_t[3];
  double prev_cost, lambda;
  double red[16 * 21];
  int hist[256];
  int cand[kLoTopK];
  int ncand, cnt, done;
};

// one locally-optimised candidate: MSAC cost at the RANSAC threshold (MAGSAC++: sum rho, in fp64) and its pose
struct LoResult {
  double cost, R[9], t[3];
};
static_assert(sizeof(LoResult) == 104 && offsetof(LoResult, cost) == 0 && offsetof(LoResult, R) == 8 &&
                  offsetof(LoResult, t) == 80,
              "LoResult layout is part of the debug interface");

// LM rounds on the Tukey-biweight M-estimator of the Sampson distance with cut-off sqrt(T2),
// starting from (S.R, S.t); leaves the last accepted parameters there. All threads must call it.
// hard = true: truncated least squares instead (weight 1 inside the cut-off, cost sum min(r^2, T2) / T2 = the MSAC cost):
// its fixed point is the least-squares optimum of the model's own inlier set.
// kScore = kMagsac: sigma-consensus++ instead, with sigma_max = sqrt(T2) (hard is ignored): the weights are the MAGSAC++
// w(r) of the current model, H = sum w J J^T, g = sum w J r (the gradient of sum rho) and the cost is sum rho, so every
// pass is one IRLS step, damped by LM. It stops after max_it passes or once sum rho drops by <= 1e-10 (relative).
template <Scoring kScore = Scoring::kMsac>
__device__ void emat_lm_round(EmatShared& S, const float4* pts, int N, double T2, int step = 1, bool hard = false,
                              int max_it = kLoInner) {
  const double sigma = kScore == Scoring::kMagsac ? sqrt(T2) : 0.0;
  if (threadIdx.x == 0) { S.lambda = 1e-6; S.prev_cost = 1e300; S.done = 0; }
  __syncthreads();
  for (int it = 0; it <= max_it; ++it) {
    if (S.done) break;   // converged: the accepted parameters are already in (prevR, prevt)
    double R[9], t[3], b1[3], b2[3];
    for (int k = 0; k < 9; ++k) R[k] = S.R[k];
    for (int k = 0; k < 3; ++k) t[k] = S.t[k];
    tangent_basis(t, b1, b2);
    double acc[21];
    for (int k = 0; k < 21; ++k) acc[k] = 0.0;
    for (int i = threadIdx.x * step; i < N; i += blockDim.x * step) {   // step > 1: every step-th correspondence
      double J[5];
      const double r = sampson_res_jac(R, t, b1, b2, pts[i], J);
      if constexpr (kScore == Scoring::kMagsac) {
        double rho, w;
        magsac_loss_sq(r * r, sigma, &rho, &w);
        if (w > 0.0) {
          int qq = 0;
          for (int a = 0; a < 5; ++a)
            for (int b = a; b < 5; ++b) acc[qq++] += w * J[a] * J[b];
          for (int a = 0; a < 5; ++a) acc[15 + a] += w * J[a] * r;
        }
        acc[20] += rho;
        continue;
      }
      const double q = r * r / T2;
      if (q < 1.0) {
        const double u = 1.0 - q, w = hard ? 1.0 : u * u;
        int qq = 0;
        for (int a = 0; a < 5; ++a)
          for (int b = a; b < 5; ++b) acc[qq++] += w * J[a] * J[b];
        for (int a = 0; a < 5; ++a) acc[15 + a] += w * J[a] * r;
        acc[20] += hard ? q : (1.0 - u * u * u);
      } else {
        acc[20] += 1.0;
      }
    }
    block_sum_256<21>(acc, S.red);
    if (threadIdx.x == 0) {
      const double cost = acc[20];
      if (cost <= S.prev_cost) {  // accept the parameters that produced this pass
        if (S.prev_cost - cost <= 1e-10 * cost) S.done = 1;   // no measurable progress any more
        S.prev_cost = cost;
        for (int k = 0; k < 9; ++k) S.prevR[k] = S.R[k];
        for (int k = 0; k < 3; ++k) S.prevt[k] = S.t[k];
        int q = 0;
        for (int a = 0; a < 5; ++a)
          for (int b = a; b < 5; ++b) { S.H[a * 5 + b] = acc[q]; S.H[b * 5 + a] = acc[q]; ++q; }
        for (int a = 0; a < 5; ++a) S.g[a] = acc[15 + a];
        S.lambda = fmax(S.lambda * 0.1, 1e-12);
      } else {                    // reject: back to the last accepted point, more damping
        S.lambda *= 10.0;
      }
      double d[5], pb1[3], pb2[3];
      tangent_basis(S.prevt, pb1, pb2);
      if (it < max_it && solve_damped(S.H, S.g, S.lambda, 5, d)) {
        double dR[9], Rn[9], tn[3];
        so3_exp(d, dR);
        mat3_mul(dR, S.prevR, Rn);
        for (int k = 0; k < 3; ++k) tn[k] = S.prevt[k] + d[3] * pb1[k] + d[4] * pb2[k];
        const double nn = norm3(tn);
        for (int k = 0; k < 9; ++k) S.R[k] = Rn[k];
        for (int k = 0; k < 3; ++k) S.t[k] = tn[k] / nn;
      } else {
        for (int k = 0; k < 9; ++k) S.R[k] = S.prevR[k];
        for (int k = 0; k < 3; ++k) S.t[k] = S.prevt[k];
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int k = 0; k < 9; ++k) S.R[k] = S.prevR[k];
    for (int k = 0; k < 3; ++k) S.t[k] = S.prevt[k];
  }
  __syncthreads();
}

// (R, t) <- the decomposition of S.E with the most points in front of both cameras among the
// correspondences with Sampson^2 < thr2 (cv.recoverPose's vote). S.cnt = that count.
__device__ void emat_choose_pose(EmatShared& S, const float4* pts, int N, double thr2) {
  if (threadIdx.x == 0) decompose_essential(S.E, S.c_R1, S.c_R2, S.c_t);
  __syncthreads();
  double cnt[4] = {0, 0, 0, 0};
  const double tn[3] = {-S.c_t[0], -S.c_t[1], -S.c_t[2]};
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float4 p = pts[i];
    if (sampson_sq(S.E, p.x, p.y, p.z, p.w) < thr2) {
      cnt[0] += cheirality_ok(S.c_R1, S.c_t, p) ? 1.0 : 0.0;
      cnt[1] += cheirality_ok(S.c_R2, S.c_t, p) ? 1.0 : 0.0;
      cnt[2] += cheirality_ok(S.c_R1, tn, p) ? 1.0 : 0.0;
      cnt[3] += cheirality_ok(S.c_R2, tn, p) ? 1.0 : 0.0;
    }
  }
  block_sum_256<4>(cnt, S.red);
  if (threadIdx.x == 0) {
    int b = 0;
    for (int k = 1; k < 4; ++k)
      if (cnt[k] > cnt[b]) b = k;
    const double* Rb = (b == 0 || b == 2) ? S.c_R1 : S.c_R2;
    for (int k = 0; k < 9; ++k) S.R[k] = Rb[k];
    for (int k = 0; k < 3; ++k) S.t[k] = (b < 2) ? S.c_t[k] : -S.c_t[k];
    S.cnt = static_cast<int>(cnt[b] + 0.5);
  }
  __syncthreads();
}

// MSAC cost (sum of min(d^2, thr2)) of the model (S.R, S.t); result broadcast to all threads
__device__ double emat_msac(EmatShared& S, const float4* pts, int N, double thr2) {
  double E[9];
  essential_from_rt(S.R, S.t, E);
  double c[1] = {0.0};
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float4 p = pts[i];
    c[0] += fmin(sampson_sq(E, p.x, p.y, p.z, p.w), thr2);
  }
  block_sum_256<1>(c, S.red);
  if (threadIdx.x == 0) S.prev_cost = c[0];
  __syncthreads();
  const double r = S.prev_cost;
  __syncthreads();
  return r;
}

// sum of the MAGSAC++ rho (sigma_max = sigma) of the model (S.R, S.t); result broadcast to all threads
__device__ double emat_sum_rho(EmatShared& S, const float4* pts, int N, double sigma) {
  double E[9];
  essential_from_rt(S.R, S.t, E);
  double c[1] = {0.0};
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float4 p = pts[i];
    double rho, w;
    magsac_loss_sq(sampson_sq(E, p.x, p.y, p.z, p.w), sigma, &rho, &w);
    c[0] += rho;
  }
  block_sum_256<1>(c, S.red);
  if (threadIdx.x == 0) S.prev_cost = c[0];
  __syncthreads();
  const double r = S.prev_cost;
  __syncthreads();
  return r;
}

// Shared prologue of the two kernels below: points of the pair into shared memory, the kLoTopK
// cheapest block winners (cheapest first) into S.cand. Returns N (0 = nothing to do).
__device__ int emat_stage_in(EmatShared& S, float4* s_pts, const float* kpts0, const float* kpts1, const int* offsets,
                             const float* K0, const float* K1, int pair, int max_pts, int blocks_per_pair,
                             const HypResult* res) {
  const int n0 = offsets[pair];
  const int N = min(offsets[pair + 1] - n0, max_pts);
  if (N < 5) return 0;
  const float* k0 = kpts0 + 2 * static_cast<size_t>(n0);
  const float* k1 = kpts1 + 2 * static_cast<size_t>(n0);
  for (int i = threadIdx.x; i < N; i += blockDim.x) s_pts[i] = normalise_pt(k0, k1, i, K0, K1);
  if (threadIdx.x == 0) {
    int n = 0;
    for (int k = 0; k < blocks_per_pair; ++k) {
      if (!res[k].valid) continue;
      int pos = n < kLoTopK ? n : kLoTopK;
      while (pos > 0 && res[S.cand[pos - 1]].cost > res[k].cost) --pos;
      if (pos >= kLoTopK) continue;
      const int last = n < kLoTopK ? n : kLoTopK - 1;
      for (int q = last; q > pos; --q) S.cand[q] = S.cand[q - 1];
      S.cand[pos] = k;
      if (n < kLoTopK) ++n;
    }
    S.ncand = n;
  }
  __syncthreads();
  return S.ncand > 0 ? N : 0;
}

// Local optimisation of ONE candidate per block: grid (pairs, kLoTopK). The candidates of a pair are
// independent, so they run on different SMs instead of one after the other.
constexpr int kLoThreads = 512;    // the LM passes are fp64-latency bound: more warps per pair
constexpr int kLoMaxPts = 1024;    // correspondences used by the candidate LO rounds (strided subsample beyond that);
                                   // the final tightening rounds and every cost / mask evaluation use all of them
// MAGSAC++ iteration caps (IRLS / LM passes; each stops earlier once sum rho drops by <= 1e-10 relative): the
// sigma-consensus++ of each candidate on the LO subsample, then the final polish of the winner on all correspondences
constexpr int kMagsacLoIters = 10, kMagsacFinalIters = 30;

template <Scoring kScore>
__global__ void __launch_bounds__(kLoThreads) emat_lo_kernel(
    const float* __restrict__ kpts0, const float* __restrict__ kpts1, const int* __restrict__ offsets,
    const float* __restrict__ K0s, const float* __restrict__ K1s, float pix_thr, int blocks_per_pair,
    int max_pts, const HypResult* __restrict__ results, LoResult* __restrict__ lo_out, int lo_enabled,
    const int* __restrict__ active) {
  extern __shared__ float4 s_pts[];
  __shared__ EmatShared S;
  const int pair = blockIdx.x, c = blockIdx.y;
  if (active && !active[pair]) return;
  LoResult* out = lo_out + static_cast<size_t>(pair) * kLoTopK + c;
  const float* K0 = K0s + 9 * pair;
  const float* K1 = K1s + 9 * pair;
  const HypResult* res = results + static_cast<size_t>(pair) * blocks_per_pair;
  const int N = emat_stage_in(S, s_pts, kpts0, kpts1, offsets, K0, K1, pair, max_pts, blocks_per_pair, res);
  if (N == 0 || c >= S.ncand || (!lo_enabled && c > 0)) {
    if (threadIdx.x == 0) out->cost = 1e300;
    return;
  }
  const double thr = static_cast<double>(emat_threshold(pix_thr, K0, K1));
  const double thr2 = thr * thr;
  if (threadIdx.x == 0)
    for (int k = 0; k < 9; ++k) S.E[k] = res[S.cand[c]].model[k];
  __syncthreads();
  emat_choose_pose(S, s_pts, N, thr2);
  if constexpr (kScore == Scoring::kMagsac) {
    emat_lm_round<Scoring::kMagsac>(S, s_pts, N, thr2, (N + kLoMaxPts - 1) / kLoMaxPts, false, kMagsacLoIters);
  } else if (lo_enabled) {
    // cut-off shrinking from 3x to 1x the RANSAC threshold
    const double sched[kLoRounds] = {3.0, 2.0, 1.5, 1.0, 1.0, 1.0};
    const int step = (N + kLoMaxPts - 1) / kLoMaxPts;
    for (int r = 0; r < kLoRounds; ++r) emat_lm_round(S, s_pts, N, sched[r] * sched[r] * thr2, step);
  }
  const double cost = kScore == Scoring::kMagsac ? emat_sum_rho(S, s_pts, N, thr) : emat_msac(S, s_pts, N, thr2);
  if (threadIdx.x == 0) {
    out->cost = cost;
    for (int k = 0; k < 9; ++k) out->R[k] = S.R[k];
    for (int k = 0; k < 3; ++k) out->t[k] = S.t[k];
  }
}

template <Scoring kScore>
__global__ void __launch_bounds__(kLoThreads) emat_final_kernel(
    const float* __restrict__ kpts0, const float* __restrict__ kpts1, const int* __restrict__ offsets,
    const float* __restrict__ K0s, const float* __restrict__ K1s, float pix_thr, int blocks_per_pair,
    int max_pts, const HypResult* __restrict__ results, const LoResult* __restrict__ lo_out,
    double* __restrict__ Rd, double* __restrict__ td,
    float* __restrict__ Rf, float* __restrict__ tf, int* __restrict__ n_inl,
    unsigned char* __restrict__ mask, int lo_enabled, const int* __restrict__ active) {
  extern __shared__ float4 s_pts[];
  __shared__ EmatShared S;
  const int pair = blockIdx.x;
  if (active && !active[pair]) return;   // a finished pair keeps R, t, n, mask, Rd and td of its last round
  const int n0 = offsets[pair];
  const int Nall = offsets[pair + 1] - n0;
  auto fail = [&]() {
    for (int i = threadIdx.x; i < Nall; i += blockDim.x) mask[n0 + i] = 0;
    if (threadIdx.x < 9) { Rf[9 * pair + threadIdx.x] = NAN; Rd[9 * pair + threadIdx.x] = NAN; }
    if (threadIdx.x < 3) { tf[3 * pair + threadIdx.x] = NAN; td[3 * pair + threadIdx.x] = NAN; }
    if (threadIdx.x == 0) n_inl[pair] = 0;
  };
  const float* K0 = K0s + 9 * pair;
  const float* K1 = K1s + 9 * pair;
  const HypResult* res = results + static_cast<size_t>(pair) * blocks_per_pair;
  const int N = emat_stage_in(S, s_pts, kpts0, kpts1, offsets, K0, K1, pair, max_pts, blocks_per_pair, res);
  if (N == 0) { fail(); return; }
  const double thr = static_cast<double>(emat_threshold(pix_thr, K0, K1));
  const double thr2 = thr * thr;
  if (threadIdx.x == 0) {
    // cheapest locally-optimised candidate, first one on ties (the order a sequential sweep would keep)
    const LoResult* lo = lo_out + static_cast<size_t>(pair) * kLoTopK;
    int bc = 0;
    for (int c = 1; c < kLoTopK; ++c)
      if (lo[c].cost < lo[bc].cost) bc = c;
    S.best_cost = lo[bc].cost;
    for (int k = 0; k < 9; ++k) S.bestR[k] = lo[bc].R[k];
    for (int k = 0; k < 3; ++k) S.bestt[k] = lo[bc].t[k];
  }
  __syncthreads();
  if (!(S.best_cost < 1e299)) { fail(); return; }
  if (threadIdx.x == 0) {
    for (int k = 0; k < 9; ++k) S.R[k] = S.bestR[k];
    for (int k = 0; k < 3; ++k) S.t[k] = S.bestt[k];
  }
  __syncthreads();
  if constexpr (kScore == Scoring::kMagsac) {
    // sigma-consensus++ polish on all correspondences; no tightening, no refit
    emat_lm_round<Scoring::kMagsac>(S, s_pts, N, thr2, 1, false, kMagsacFinalIters);
  } else if (lo_enabled) {
    // noise-adaptive tightening: robust scale of the inlier residuals (1.4826 * median |r|), cut-off
    // = clamp(3 sigma, ., thr). With clean data this discards chance near-threshold outliers that a
    // fixed cut-off keeps (the sigma-consensus idea of MAGSAC++).
    for (int round = 0; round < kTightRounds; ++round) {
      for (int k = threadIdx.x; k < 256; k += blockDim.x) S.hist[k] = 0;
      __syncthreads();
      double E[9];
      essential_from_rt(S.R, S.t, E);
      for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const float4 p = s_pts[i];
        const double d2 = sampson_sq(E, p.x, p.y, p.z, p.w);
        if (d2 < thr2) atomicAdd(&S.hist[min(255, static_cast<int>(sqrt(d2 / thr2) * 256.0))], 1);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        int tot = 0;
        for (int k = 0; k < 256; ++k) tot += S.hist[k];
        int acc = 0, med = 255;
        for (int k = 0; k < 256; ++k) {
          acc += S.hist[k];
          if (2 * acc >= tot) { med = k; break; }
        }
        const double sigma = 1.4826 * (med + 1) / 256.0 * thr;
        S.lambda = fmin(thr, fmax(3.0 * sigma, 0.02 * thr));  // cut-off for this round
      }
      __syncthreads();
      const double T = S.lambda;
      __syncthreads();
      emat_lm_round(S, s_pts, N, T * T);
    }
    // safeguard: keep the pre-tightening model if tightening made the MSAC cost at thr worse by > 2 %
    const double cost = emat_msac(S, s_pts, N, thr2);
    if (threadIdx.x == 0 && cost > 1.02 * S.best_cost) {
      for (int k = 0; k < 9; ++k) S.R[k] = S.bestR[k];
      for (int k = 0; k < 3; ++k) S.t[k] = S.bestt[k];
    }
    __syncthreads();
    if (lo_enabled & 2) {
      // reference-equivalent refit (SURVEY §7 hard part 1(b)): truncated least squares at the RANSAC threshold, i.e. LM
      // on the MSAC cost, whose fixed point is the Sampson least-squares optimum of the model's OWN inlier set — the
      // point the "polished oracle" (OpenCV's mask -> Sampson LM, oracle/pose_solver_oracle.py) sits at.
      for (int round = 0; round < 4; ++round) emat_lm_round(S, s_pts, N, thr2, 1, true, 8);
    }
  }
  if (threadIdx.x == 0) essential_from_rt(S.R, S.t, S.E);
  __syncthreads();
  // ---- final mask: Sampson^2 < thr^2 under the final E (what cv.findEssentialMat returns), then
  // the cheirality filter that cv.recoverPose applies to the mask in place (pose_solver.py:57)
  emat_choose_pose(S, s_pts, N, thr2);
  double cnt[1] = {0.0};
  for (int i = threadIdx.x; i < Nall; i += blockDim.x) {
    unsigned char m = 0;
    if (i < N) {
      const float4 p = s_pts[i];
      if (sampson_sq(S.E, p.x, p.y, p.z, p.w) < thr2 && cheirality_ok(S.R, S.t, p)) m = 1;
    }
    mask[n0 + i] = m;
    cnt[0] += m;
  }
  block_sum_256<1>(cnt, S.red);
  if (threadIdx.x == 0) S.cnt = static_cast<int>(cnt[0] + 0.5);
  __syncthreads();
  if (S.cnt == 0) { fail(); return; }
  if (threadIdx.x < 9) { Rd[9 * pair + threadIdx.x] = S.R[threadIdx.x]; Rf[9 * pair + threadIdx.x] = static_cast<float>(S.R[threadIdx.x]); }
  if (threadIdx.x < 3) { td[3 * pair + threadIdx.x] = S.t[threadIdx.x]; tf[3 * pair + threadIdx.x] = static_cast<float>(S.t[threadIdx.x]); }
  if (threadIdx.x == 0) n_inl[pair] = S.cnt;
}

// ================================================================================================
// scale from depth (EssentialMatrixMetricSolver, pose_solver.py:132-172)
// ================================================================================================
__device__ __forceinline__ void inverse_K_f32(const float* K, float* Ki) {
  // np.linalg.inv on the float32 intrinsics; adjugate in double, rounded to float32
  double A[9];
  for (int k = 0; k < 9; ++k) A[k] = K[k];
  const double d = det3(A);
  const double inv[9] = {
      (A[4] * A[8] - A[5] * A[7]) / d, (A[2] * A[7] - A[1] * A[8]) / d, (A[1] * A[5] - A[2] * A[4]) / d,
      (A[5] * A[6] - A[3] * A[8]) / d, (A[0] * A[8] - A[2] * A[6]) / d, (A[2] * A[3] - A[0] * A[5]) / d,
      (A[3] * A[7] - A[4] * A[6]) / d, (A[1] * A[6] - A[0] * A[7]) / d, (A[0] * A[4] - A[1] * A[3]) / d};
  for (int k = 0; k < 9; ++k) Ki[k] = static_cast<float>(inv[k]);
}

__device__ __forceinline__ void backproject(const float* Ki, int u, int v, float depth, double* xyz) {
  const double d = depth;
  for (int r = 0; r < 3; ++r)
    xyz[r] = d * (static_cast<double>(Ki[3 * r]) * u + static_cast<double>(Ki[3 * r + 1]) * v +
                  static_cast<double>(Ki[3 * r + 2]));
}

__global__ void __launch_bounds__(1024) scale_consensus_kernel(
    const float* __restrict__ kpts0, const float* __restrict__ kpts1, const int* __restrict__ offsets,
    const float* __restrict__ K0s, const float* __restrict__ K1s, const unsigned char* __restrict__ mask,
    const double* __restrict__ Rd, const double* __restrict__ td, const float* __restrict__ depth0,
    const float* __restrict__ depth1, int H, int W, double scale_thr, int max_pts, float* __restrict__ R_out,
    float* __restrict__ t_out, int* __restrict__ inl_out) {
  extern __shared__ double s_scale[];
  __shared__ int s_bc[32], s_bi[32];
  __shared__ float s_Ki0[9], s_Ki1[9];
  const int pair = blockIdx.x;
  const int n0 = offsets[pair];
  const int N = min(offsets[pair + 1] - n0, max_pts);
  const double* R = Rd + 9 * pair;
  const double* t = td + 3 * pair;
  if (threadIdx.x == 0) {
    inverse_K_f32(K0s + 9 * pair, s_Ki0);
    inverse_K_f32(K1s + 9 * pair, s_Ki1);
  }
  __syncthreads();
  const bool pose_ok = (R[0] == R[0]) && (t[0] == t[0]);
  const float* d0 = depth0 + static_cast<size_t>(pair) * H * W;
  const float* d1 = depth1 + static_cast<size_t>(pair) * H * W;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    double s = NAN;
    if (pose_ok && mask[n0 + i]) {
      int u0 = static_cast<int>(kpts0[2 * (n0 + i)]), v0 = static_cast<int>(kpts0[2 * (n0 + i) + 1]);
      int u1 = static_cast<int>(kpts1[2 * (n0 + i)]), v1 = static_cast<int>(kpts1[2 * (n0 + i) + 1]);
      if (u0 >= 0 && u0 < W && v0 >= 0 && v0 < H && u1 >= 0 && u1 < W && v1 >= 0 && v1 < H) {
        const float z0 = d0[v0 * W + u0], z1 = d1[v1 * W + u1];
        if (z0 > 0.f && z1 > 0.f) {
          double X0[3], X1[3], RX0[3];
          backproject(s_Ki0, u0, v0, z0, X0);
          backproject(s_Ki1, u1, v1, z1, X1);
          mat3_vec(R, X0, RX0);
          s = (X1[0] - RX0[0]) * t[0] + (X1[1] - RX0[1]) * t[1] + (X1[2] - RX0[2]) * t[2];
        }
      }
    }
    s_scale[i] = s;
  }
  __syncthreads();
  // exhaustive consensus, strict '<', first best wins (pose_solver.py:160-166)
  int bc = 0, bi = 0x7fffffff;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const double si = s_scale[i];
    if (!(si == si)) continue;
    int c = 0;
    for (int j = 0; j < N; ++j) c += (fabs(s_scale[j] - si) < scale_thr) ? 1 : 0;
    if (c > bc) { bc = c; bi = i; }
  }
  // block arg-max (count desc, index asc)
  for (int o = 16; o > 0; o >>= 1) {
    const int oc = __shfl_xor_sync(0xffffffffu, bc, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (oc > bc || (oc == bc && oi < bi)) { bc = oc; bi = oi; }
  }
  if ((threadIdx.x & 31) == 0) { s_bc[threadIdx.x >> 5] = bc; s_bi[threadIdx.x >> 5] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 32; ++w)
      if (s_bc[w] > bc || (s_bc[w] == bc && s_bi[w] < bi)) { bc = s_bc[w]; bi = s_bi[w]; }
    if (bc > 0) {
      const double s = s_scale[bi];
      for (int k = 0; k < 9; ++k) R_out[9 * pair + k] = static_cast<float>(R[k]);
      for (int k = 0; k < 3; ++k) t_out[3 * pair + k] = static_cast<float>(s * t[k]);
      inl_out[pair] = bc;
    } else {
      for (int k = 0; k < 9; ++k) R_out[9 * pair + k] = NAN;
      for (int k = 0; k < 3; ++k) t_out[3 * pair + k] = NAN;
      inl_out[pair] = 0;
    }
  }
}

// ================================================================================================
// PnP (pose_solver.py:184-235)
// ================================================================================================
__global__ void depth_min_kernel(const float* __restrict__ depth, long long hw, unsigned int* __restrict__ dmin) {
  const int pair = blockIdx.y;
  const float* d = depth + static_cast<size_t>(pair) * hw;
  float m = 3.0e38f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < hw;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    m = fminf(m, d[i]);
  for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMin(dmin + pair, __float_as_uint(fmaxf(m, 0.f)));
}

// ordered compaction of the depth-valid correspondences of each pair + 3-D lift in camera 0
__global__ void __launch_bounds__(1024) pnp_prepare_kernel(
    const float* __restrict__ kpts0, const float* __restrict__ kpts1, const int* __restrict__ offsets,
    const float* __restrict__ K0s, const float* __restrict__ depth0, int H, int W,
    const unsigned int* __restrict__ dmin, int max_pts, double* __restrict__ Xw, float* __restrict__ uv,
    int* __restrict__ vidx, int* __restrict__ nvalid) {
  __shared__ int wsum[32];
  __shared__ int base;
  __shared__ float s_Ki[9];
  const int pair = blockIdx.x;
  const int n0 = offsets[pair];
  const int N = min(offsets[pair + 1] - n0, max_pts);
  if (threadIdx.x == 0) { base = 0; inverse_K_f32(K0s + 9 * pair, s_Ki); }
  __syncthreads();
  const float dm = __uint_as_float(dmin[pair]);
  const float* d0 = depth0 + static_cast<size_t>(pair) * H * W;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int i0 = 0; i0 < N; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    int flag = 0, u = 0, v = 0;
    float z = 0.f;
    if (i < N) {
      u = static_cast<int>(kpts0[2 * (n0 + i)]);
      v = static_cast<int>(kpts0[2 * (n0 + i) + 1]);
      if (u >= 0 && u < W && v >= 0 && v < H) {
        z = d0[v * W + u];
        flag = z > dm ? 1 : 0;
      }
    }
    int inc = flag;
    for (int o = 1; o < 32; o <<= 1) {
      const int tt = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += tt;
    }
    if (lane == 31) wsum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      int w = wsum[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const int tt = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += tt;
      }
      wsum[lane] = w;
    }
    __syncthreads();
    if (flag) {
      const int slot = pair * max_pts + base + (wid > 0 ? wsum[wid - 1] : 0) + inc - 1;
      double X[3];
      backproject(s_Ki, u, v, z, X);
      Xw[3 * slot] = X[0]; Xw[3 * slot + 1] = X[1]; Xw[3 * slot + 2] = X[2];
      uv[2 * slot] = kpts1[2 * (n0 + i)];
      uv[2 * slot + 1] = kpts1[2 * (n0 + i) + 1];
      vidx[slot] = i;
    }
    __syncthreads();
    if (threadIdx.x == 0) base += wsum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) nvalid[pair] = base;
}

struct PnpPt { float X, Y, Z, u, v; };

__global__ void __launch_bounds__(kHypPerBlock) pnp_hyp_kernel(
    const double* __restrict__ Xw, const float* __restrict__ uv, const int* __restrict__ offsets,
    const int* __restrict__ nvalid, const float* __restrict__ K1s, float reproj_thr, int num_hyp,
    unsigned long long seed, int max_pts, HypResult* __restrict__ results, const int* __restrict__ active) {
  extern __shared__ float s_raw[];
  __shared__ HypResult s_best[kHypPerBlock / 32];
  const int pair = blockIdx.y;
  if (active && !active[pair]) return;
  const int s0 = pair * max_pts;   // scratch rows of this pair (compacted, at most max_pts)
  const int N = nvalid[pair];
  HypResult* out = results + static_cast<size_t>(pair) * gridDim.x + blockIdx.x;
  if (N < 4) {
    if (threadIdx.x == 0) { out->valid = 0; out->cost = 1e300; out->count = 0; }
    return;
  }
  float* sX = s_raw;            // [N][3]
  float* sU = s_raw + 3 * N;    // [N][2]
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    sX[3 * i] = static_cast<float>(Xw[3 * (s0 + i)]);
    sX[3 * i + 1] = static_cast<float>(Xw[3 * (s0 + i) + 1]);
    sX[3 * i + 2] = static_cast<float>(Xw[3 * (s0 + i) + 2]);
    sU[2 * i] = uv[2 * (s0 + i)];
    sU[2 * i + 1] = uv[2 * (s0 + i) + 1];
  }
  __syncthreads();
  const float* K1 = K1s + 9 * pair;
  const float fx = K1[0], fy = K1[4], cx = K1[2], cy = K1[5];
  const float thr2 = reproj_thr * reproj_thr;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.x * kHypPerBlock + threadIdx.x;
  double Rm[9], tm[3];
  int have = 0;
  if (h < num_hyp) {
    unsigned long long st = seed ^ (0xA24BAED4963EE407ull * (static_cast<unsigned long long>(pair) + 1)) ^
                            (0x9E3779B97F4A7C15ull * (static_cast<unsigned long long>(h) + 1));
    int idx[4];
    sample_distinct<4>(st, N, idx);
    double X[3][3], f[3][3];
    for (int k = 0; k < 3; ++k) {
      for (int c = 0; c < 3; ++c) X[k][c] = Xw[3 * (s0 + idx[k]) + c];
      const double bx = (static_cast<double>(uv[2 * (s0 + idx[k])]) - cx) / fx;
      const double by = (static_cast<double>(uv[2 * (s0 + idx[k]) + 1]) - cy) / fy;
      const double nn = 1.0 / sqrt(bx * bx + by * by + 1.0);
      f[k][0] = bx * nn; f[k][1] = by * nn; f[k][2] = nn;
    }
    double Rs[4][9], ts[4][3];
    const int ns = p3p(X, f, Rs, ts);
    // disambiguate with the 4th point (what cv's P3P does with 4 input points)
    double best = 1e300;
    const double X4[3] = {Xw[3 * (s0 + idx[3])], Xw[3 * (s0 + idx[3]) + 1], Xw[3 * (s0 + idx[3]) + 2]};
    const double u4 = uv[2 * (s0 + idx[3])], v4 = uv[2 * (s0 + idx[3]) + 1];
    for (int s = 0; s < ns; ++s) {
      double Xc[3];
      mat3_vec(Rs[s], X4, Xc);
      for (int c = 0; c < 3; ++c) Xc[c] += ts[s][c];
      if (!(Xc[2] > 1e-9)) continue;
      const double du = fx * Xc[0] / Xc[2] + cx - u4, dv = fy * Xc[1] / Xc[2] + cy - v4;
      const double e = du * du + dv * dv;
      if (e < best) {
        best = e;
        have = 1;
        for (int c = 0; c < 9; ++c) Rm[c] = Rs[s][c];
        for (int c = 0; c < 3; ++c) tm[c] = ts[s][c];
      }
    }
  }
  int best_cnt = -1, best_src = -1;
  for (int src = 0; src < 32; ++src) {
    if (!__shfl_sync(0xffffffffu, have, src)) continue;
    float R[9], t[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = __shfl_sync(0xffffffffu, static_cast<float>(Rm[k]), src);
#pragma unroll
    for (int k = 0; k < 3; ++k) t[k] = __shfl_sync(0xffffffffu, static_cast<float>(tm[k]), src);
    int inl = 0;
    for (int i0 = 0; i0 < N; i0 += 32) {
      const int i = i0 + lane;
      bool ok = false;
      if (i < N) {
        const float X = sX[3 * i], Y = sX[3 * i + 1], Z = sX[3 * i + 2];
        const float xc = fmaf(R[0], X, fmaf(R[1], Y, fmaf(R[2], Z, t[0])));
        const float yc = fmaf(R[3], X, fmaf(R[4], Y, fmaf(R[5], Z, t[1])));
        const float zc = fmaf(R[6], X, fmaf(R[7], Y, fmaf(R[8], Z, t[2])));
        if (zc > 1e-6f) {
          const float iz = 1.f / zc;
          const float du = fmaf(fx * xc, iz, cx) - sU[2 * i], dv = fmaf(fy * yc, iz, cy) - sU[2 * i + 1];
          ok = fmaf(du, du, dv * dv) < thr2;
        }
      }
      inl += __popc(__ballot_sync(0xffffffffu, ok));
    }
    if (inl > best_cnt) { best_cnt = inl; best_src = src; }
  }
  if (lane == 0) {
    s_best[warp].valid = best_src >= 0 ? 1 : 0;
    s_best[warp].cost = best_src >= 0 ? -static_cast<double>(best_cnt) : 1e300;
    s_best[warp].count = best_cnt;
  }
  if (best_src >= 0 && lane == best_src) {
    for (int k = 0; k < 9; ++k) s_best[warp].model[k] = Rm[k];
    for (int k = 0; k < 3; ++k) s_best[warp].model[9 + k] = tm[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int bw = 0;
    for (int w = 1; w < kHypPerBlock / 32; ++w)
      if (s_best[w].cost < s_best[bw].cost) bw = w;
    *out = s_best[bw];
  }
}

constexpr int kPnpIters = 20;

__global__ void __launch_bounds__(256) pnp_final_kernel(
    const double* __restrict__ Xw, const float* __restrict__ uv, const int* __restrict__ vidx,
    const int* __restrict__ offsets, const int* __restrict__ nvalid, const float* __restrict__ K1s,
    float reproj_thr, int blocks_per_pair, int max_pts, const HypResult* __restrict__ results, float* __restrict__ Rf,
    float* __restrict__ tf, int* __restrict__ n_inl, unsigned char* __restrict__ mask, const int* __restrict__ active) {
  __shared__ double sh_red[8 * 28];
  __shared__ double s_R[9], s_t[3], s_R0[9], s_t0[3], s_prevR[9], s_prevt[3], s_H[36], s_g[6];
  __shared__ double s_prev_cost, s_lambda;
  __shared__ int s_flag, s_n;
  const int pair = blockIdx.x;
  if (active && !active[pair]) return;   // a finished pair keeps R, t, n and mask of its last round
  const int n0 = offsets[pair];
  const int Nall = offsets[pair + 1] - n0;
  const int s0 = pair * max_pts;
  const int N = nvalid[pair];
  for (int i = threadIdx.x; i < Nall; i += blockDim.x) mask[n0 + i] = 0;
  auto fail = [&]() {
    if (threadIdx.x < 9) Rf[9 * pair + threadIdx.x] = NAN;
    if (threadIdx.x < 3) tf[3 * pair + threadIdx.x] = NAN;
    if (threadIdx.x == 0) n_inl[pair] = 0;
  };
  if (threadIdx.x == 0) {
    int b = -1;
    if (N >= 4) {
      const HypResult* r = results + static_cast<size_t>(pair) * blocks_per_pair;
      for (int k = 0; k < blocks_per_pair; ++k)
        if (r[k].valid && (b < 0 || r[k].cost < r[b].cost)) b = k;
      if (b >= 0) {
        for (int k = 0; k < 9; ++k) { s_R[k] = r[b].model[k]; s_R0[k] = s_R[k]; }
        for (int k = 0; k < 3; ++k) { s_t[k] = r[b].model[9 + k]; s_t0[k] = s_t[k]; }
      }
    }
    s_flag = b;
  }
  __syncthreads();
  if (s_flag < 0) { fail(); return; }
  const float* K1 = K1s + 9 * pair;
  const double fx = K1[0], fy = K1[4], cx = K1[2], cy = K1[5];
  const double thr2 = static_cast<double>(reproj_thr) * reproj_thr;
  __syncthreads();
  // inlier set of the RANSAC model (fixed during the refinement, like cv.solvePnPRansac's)
  auto is_inlier = [&](int i) {
    const double* X = Xw + 3 * (s0 + i);
    double Xc[3];
    mat3_vec(s_R0, X, Xc);
    for (int c = 0; c < 3; ++c) Xc[c] += s_t0[c];
    if (!(Xc[2] > 1e-9)) return false;
    const double du = fx * Xc[0] / Xc[2] + cx - uv[2 * (s0 + i)], dv = fy * Xc[1] / Xc[2] + cy - uv[2 * (s0 + i) + 1];
    return du * du + dv * dv < thr2;
  };
  double cnt[1] = {0.0};
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    if (is_inlier(i)) { cnt[0] += 1.0; mask[n0 + vidx[s0 + i]] = 1; }
  block_sum_256<1>(cnt, sh_red);
  if (threadIdx.x == 0) { s_n = static_cast<int>(cnt[0] + 0.5); s_lambda = 1e-6; s_prev_cost = 1e300; }
  __syncthreads();
  const int n_in = s_n;
  if (n_in < 4) { fail(); for (int i = threadIdx.x; i < Nall; i += blockDim.x) mask[n0 + i] = 0; return; }
  if (n_in >= 6) {  // LM refinement on the inliers (pose_solver.py:216-220)
    for (int it = 0; it <= kPnpIters; ++it) {
      double R[9], t[3];
      for (int k = 0; k < 9; ++k) R[k] = s_R[k];
      for (int k = 0; k < 3; ++k) t[k] = s_t[k];
      double acc[28];
      for (int k = 0; k < 28; ++k) acc[k] = 0.0;
      for (int i = threadIdx.x; i < N; i += blockDim.x) {
        if (!is_inlier(i)) continue;
        const double* X = Xw + 3 * (s0 + i);
        double RX[3], Xc[3];
        mat3_vec(R, X, RX);
        for (int c = 0; c < 3; ++c) Xc[c] = RX[c] + t[c];
        const double iz = 1.0 / Xc[2];
        const double ru = fx * Xc[0] * iz + cx - uv[2 * (s0 + i)];
        const double rv = fy * Xc[1] * iz + cy - uv[2 * (s0 + i) + 1];
        // d(u,v)/dXc
        const double a0 = fx * iz, a2 = -fx * Xc[0] * iz * iz, b1 = fy * iz, b2 = -fy * Xc[1] * iz * iz;
        // dXc/d(omega) = -[RX]x ; dXc/dt = I
        double Ju[6], Jv[6];
        Ju[0] = a2 * RX[1];                 // a . (e0 x RX) = a0*0 + 0 + a2*( RX[1]) ... see below
        Ju[1] = a0 * RX[2] - a2 * RX[0];
        Ju[2] = -a0 * RX[1];
        Jv[0] = -b1 * RX[2] + b2 * RX[1];
        Jv[1] = -b2 * RX[0];
        Jv[2] = b1 * RX[0];
        Ju[3] = a0; Ju[4] = 0.0; Ju[5] = a2;
        Jv[3] = 0.0; Jv[4] = b1; Jv[5] = b2;
        int q = 0;
        for (int a = 0; a < 6; ++a)
          for (int b = a; b < 6; ++b) acc[q++] += Ju[a] * Ju[b] + Jv[a] * Jv[b];
        for (int a = 0; a < 6; ++a) acc[21 + a] += Ju[a] * ru + Jv[a] * rv;
        acc[27] += ru * ru + rv * rv;
      }
      block_sum_256<28>(acc, sh_red);
      if (threadIdx.x == 0) {
        const double cost = acc[27];
        if (cost <= s_prev_cost) {
          s_prev_cost = cost;
          for (int k = 0; k < 9; ++k) s_prevR[k] = s_R[k];
          for (int k = 0; k < 3; ++k) s_prevt[k] = s_t[k];
          int q = 0;
          for (int a = 0; a < 6; ++a)
            for (int b = a; b < 6; ++b) { s_H[a * 6 + b] = acc[q]; s_H[b * 6 + a] = acc[q]; ++q; }
          for (int a = 0; a < 6; ++a) s_g[a] = acc[21 + a];
          s_lambda = fmax(s_lambda * 0.1, 1e-12);
        } else {
          s_lambda *= 10.0;
        }
        double d[6];
        if (it < kPnpIters && solve_damped(s_H, s_g, s_lambda, 6, d)) {
          double dR[9], Rn[9];
          so3_exp(d, dR);
          mat3_mul(dR, s_prevR, Rn);
          for (int k = 0; k < 9; ++k) s_R[k] = Rn[k];
          for (int k = 0; k < 3; ++k) s_t[k] = s_prevt[k] + d[3 + k];
        } else {
          for (int k = 0; k < 9; ++k) s_R[k] = s_prevR[k];
          for (int k = 0; k < 3; ++k) s_t[k] = s_prevt[k];
        }
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      for (int k = 0; k < 9; ++k) s_R[k] = s_prevR[k];
      for (int k = 0; k < 3; ++k) s_t[k] = s_prevt[k];
    }
    __syncthreads();
  }
  const double tn = sqrt(s_t[0] * s_t[0] + s_t[1] * s_t[1] + s_t[2] * s_t[2]);
  if (!(tn <= 1000.0)) {  // pose_solver.py:223-225
    fail();
    for (int i = threadIdx.x; i < Nall; i += blockDim.x) mask[n0 + i] = 0;
    return;
  }
  if (threadIdx.x < 9) Rf[9 * pair + threadIdx.x] = static_cast<float>(s_R[threadIdx.x]);
  if (threadIdx.x < 3) tf[3 * pair + threadIdx.x] = static_cast<float>(s_t[threadIdx.x]);
  if (threadIdx.x == 0) n_inl[pair] = n_in;
}


// ================================================================================================
// Procrustes (pose_solver.py:238-320, REFINE = False): 3-D/3-D correspondences from both depth maps,
// RANSAC over 3-point Kabsch alignments, refit on the inliers. (The reference delegates this to
// Open3D's registration_ransac_based_on_correspondence.)
// ================================================================================================
// kabsch_from_sums (geometry_solvers.cuh, host hook mfr_host_kabsch): R, t from the moment sums of the inliers
__global__ void __launch_bounds__(1024) procrustes_prepare_kernel(
    const float* __restrict__ kpts0, const float* __restrict__ kpts1, const int* __restrict__ offsets,
    const float* __restrict__ K0s, const float* __restrict__ K1s, const float* __restrict__ depth0,
    const float* __restrict__ depth1, int H, int W, const unsigned int* __restrict__ dmin0,
    const unsigned int* __restrict__ dmin1, int max_pts, double* __restrict__ X0, double* __restrict__ X1,
    int* __restrict__ nvalid) {
  __shared__ int wsum[32];
  __shared__ int base;
  __shared__ float s_Ki0[9], s_Ki1[9];
  const int pair = blockIdx.x;
  const int n0 = offsets[pair];
  const int N = min(offsets[pair + 1] - n0, max_pts);
  if (threadIdx.x == 0) { base = 0; inverse_K_f32(K0s + 9 * pair, s_Ki0); inverse_K_f32(K1s + 9 * pair, s_Ki1); }
  __syncthreads();
  const float m0 = __uint_as_float(dmin0[pair]), m1 = __uint_as_float(dmin1[pair]);
  const float* d0 = depth0 + static_cast<size_t>(pair) * H * W;
  const float* d1 = depth1 + static_cast<size_t>(pair) * H * W;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int i0 = 0; i0 < N; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    int flag = 0, u0 = 0, v0 = 0, u1 = 0, v1 = 0;
    float z0 = 0.f, z1 = 0.f;
    if (i < N) {
      u0 = static_cast<int>(kpts0[2 * (n0 + i)]); v0 = static_cast<int>(kpts0[2 * (n0 + i) + 1]);
      u1 = static_cast<int>(kpts1[2 * (n0 + i)]); v1 = static_cast<int>(kpts1[2 * (n0 + i) + 1]);
      if (u0 >= 0 && u0 < W && v0 >= 0 && v0 < H && u1 >= 0 && u1 < W && v1 >= 0 && v1 < H) {
        z0 = d0[v0 * W + u0]; z1 = d1[v1 * W + u1];
        flag = (z0 > m0 && z1 > m1) ? 1 : 0;       // pose_solver.py:261
      }
    }
    int inc = flag;
    for (int o = 1; o < 32; o <<= 1) {
      const int tt = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += tt;
    }
    if (lane == 31) wsum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      int w = wsum[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const int tt = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += tt;
      }
      wsum[lane] = w;
    }
    __syncthreads();
    if (flag) {
      const int slot = pair * max_pts + base + (wid > 0 ? wsum[wid - 1] : 0) + inc - 1;
      double A[3], Bq[3];
      backproject(s_Ki0, u0, v0, z0, A);
      backproject(s_Ki1, u1, v1, z1, Bq);
      for (int k = 0; k < 3; ++k) { X0[3 * slot + k] = A[k]; X1[3 * slot + k] = Bq[k]; }
    }
    __syncthreads();
    if (threadIdx.x == 0) base += wsum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) nvalid[pair] = base;
}

__global__ void __launch_bounds__(kHypPerBlock) procrustes_hyp_kernel(
    const double* __restrict__ X0, const double* __restrict__ X1, const int* __restrict__ offsets,
    const int* __restrict__ nvalid, float max_dist, int num_hyp, unsigned long long seed, int max_pts,
    HypResult* __restrict__ results) {
  extern __shared__ float s_raw[];
  __shared__ HypResult s_best[kHypPerBlock / 32];
  const int pair = blockIdx.y;
  const size_t n0 = static_cast<size_t>(pair) * max_pts;   // scratch rows of this pair
  const int N = nvalid[pair];
  HypResult* out = results + static_cast<size_t>(pair) * gridDim.x + blockIdx.x;
  if (N < 3) {
    if (threadIdx.x == 0) { out->valid = 0; out->cost = 1e300; out->count = 0; }
    return;
  }
  float* sP = s_raw;          // [N][3]
  float* sQ = s_raw + 3 * N;  // [N][3]
  for (int i = threadIdx.x; i < 3 * N; i += blockDim.x) {
    sP[i] = static_cast<float>(X0[3 * static_cast<size_t>(n0) + i]);
    sQ[i] = static_cast<float>(X1[3 * static_cast<size_t>(n0) + i]);
  }
  __syncthreads();
  const float thr2 = max_dist * max_dist;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int h = blockIdx.x * kHypPerBlock + threadIdx.x;
  double Rm[9], tm[3];
  int have = 0;
  if (h < num_hyp) {
    unsigned long long st = seed ^ (0xC2B2AE3D27D4EB4Full * (static_cast<unsigned long long>(pair) + 1)) ^
                            (0x9E3779B97F4A7C15ull * (static_cast<unsigned long long>(h) + 1));
    int idx[3];
    sample_distinct<3>(st, N, idx);
    double sp[3] = {0, 0, 0}, sq[3] = {0, 0, 0}, spq[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = 0; k < 3; ++k) {
      const double* pp = X0 + 3 * (static_cast<size_t>(n0) + idx[k]);
      const double* qq = X1 + 3 * (static_cast<size_t>(n0) + idx[k]);
      for (int a = 0; a < 3; ++a) {
        sp[a] += pp[a]; sq[a] += qq[a];
        for (int b = 0; b < 3; ++b) spq[3 * a + b] += pp[a] * qq[b];
      }
    }
    have = kabsch_from_sums(3.0, sp, sq, spq, Rm, tm) ? 1 : 0;
  }
  int best_cnt = -1, best_src = -1;
  float best_err = 3.0e38f;
  for (int src = 0; src < 32; ++src) {
    if (!__shfl_sync(0xffffffffu, have, src)) continue;
    float R[9], t[3];
#pragma unroll
    for (int k = 0; k < 9; ++k) R[k] = __shfl_sync(0xffffffffu, static_cast<float>(Rm[k]), src);
#pragma unroll
    for (int k = 0; k < 3; ++k) t[k] = __shfl_sync(0xffffffffu, static_cast<float>(tm[k]), src);
    int inl = 0;
    float err = 0.f;
    for (int i0 = 0; i0 < N; i0 += 32) {
      const int i = i0 + lane;
      bool ok = false;
      if (i < N) {
        const float X = sP[3 * i], Y = sP[3 * i + 1], Z = sP[3 * i + 2];
        const float dx = fmaf(R[0], X, fmaf(R[1], Y, fmaf(R[2], Z, t[0]))) - sQ[3 * i];
        const float dy = fmaf(R[3], X, fmaf(R[4], Y, fmaf(R[5], Z, t[1]))) - sQ[3 * i + 1];
        const float dz = fmaf(R[6], X, fmaf(R[7], Y, fmaf(R[8], Z, t[2]))) - sQ[3 * i + 2];
        const float d2 = fmaf(dx, dx, fmaf(dy, dy, dz * dz));
        ok = d2 < thr2;
        if (ok) err += d2;
      }
      inl += __popc(__ballot_sync(0xffffffffu, ok));
    }
    err = warp_sum_f(err);
    if (inl > best_cnt || (inl == best_cnt && err < best_err)) { best_cnt = inl; best_err = err; best_src = src; }
  }
  if (lane == 0) {
    s_best[warp].valid = best_src >= 0 ? 1 : 0;
    s_best[warp].cost = best_src >= 0 ? -static_cast<double>(best_cnt) + 1e-9 * best_err : 1e300;
    s_best[warp].count = best_cnt;
  }
  if (best_src >= 0 && lane == best_src) {
    for (int k = 0; k < 9; ++k) s_best[warp].model[k] = Rm[k];
    for (int k = 0; k < 3; ++k) s_best[warp].model[9 + k] = tm[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int bw = 0;
    for (int w = 1; w < kHypPerBlock / 32; ++w)
      if (s_best[w].cost < s_best[bw].cost) bw = w;
    *out = s_best[bw];
  }
}

__global__ void __launch_bounds__(256) procrustes_final_kernel(
    const double* __restrict__ X0, const double* __restrict__ X1, const int* __restrict__ offsets,
    const int* __restrict__ nvalid, float max_dist, int blocks_per_pair, int max_pts, const HypResult* __restrict__ results,
    float* __restrict__ Rf, float* __restrict__ tf, int* __restrict__ n_inl) {
  __shared__ double sh_red[8 * 16];
  __shared__ double s_R[9], s_t[3];
  __shared__ int s_flag, s_cnt;
  const int pair = blockIdx.x;
  const size_t n0 = static_cast<size_t>(pair) * max_pts;   // scratch rows of this pair
  const int N = nvalid[pair];
  auto fail = [&]() {
    if (threadIdx.x < 9) Rf[9 * pair + threadIdx.x] = NAN;
    if (threadIdx.x < 3) tf[3 * pair + threadIdx.x] = NAN;
    if (threadIdx.x == 0) n_inl[pair] = 0;
  };
  if (threadIdx.x == 0) {
    int b = -1;
    if (N >= 3) {
      const HypResult* r = results + static_cast<size_t>(pair) * blocks_per_pair;
      for (int k = 0; k < blocks_per_pair; ++k)
        if (r[k].valid && (b < 0 || r[k].cost < r[b].cost)) b = k;
      if (b >= 0) {
        for (int k = 0; k < 9; ++k) s_R[k] = r[b].model[k];
        for (int k = 0; k < 3; ++k) s_t[k] = r[b].model[9 + k];
      }
    }
    s_flag = b;
  }
  __syncthreads();
  if (s_flag < 0) { fail(); return; }
  const double thr2 = static_cast<double>(max_dist) * max_dist;
  // refit on the inliers of the current model, re-select, twice (Open3D re-estimates on the inliers)
  for (int round = 0; round < 3; ++round) {
    double acc[16];
    for (int k = 0; k < 16; ++k) acc[k] = 0.0;
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
      const double* p = X0 + 3 * (static_cast<size_t>(n0) + i);
      const double* q = X1 + 3 * (static_cast<size_t>(n0) + i);
      double Rp[3];
      mat3_vec(s_R, p, Rp);
      const double dx = Rp[0] + s_t[0] - q[0], dy = Rp[1] + s_t[1] - q[1], dz = Rp[2] + s_t[2] - q[2];
      if (dx * dx + dy * dy + dz * dz < thr2) {
        acc[0] += 1.0;
        for (int a = 0; a < 3; ++a) {
          acc[1 + a] += p[a]; acc[4 + a] += q[a];
          for (int b = 0; b < 3; ++b) acc[7 + 3 * a + b] += p[a] * q[b];
        }
      }
    }
    block_sum_256<16>(acc, sh_red);
    if (threadIdx.x == 0) {
      s_cnt = static_cast<int>(acc[0] + 0.5);
      if (round < 2) {
        double R[9], t[3];
        if (kabsch_from_sums(acc[0], acc + 1, acc + 4, acc + 7, R, t)) {
          for (int k = 0; k < 9; ++k) s_R[k] = R[k];
          for (int k = 0; k < 3; ++k) s_t[k] = t[k];
        }
      }
    }
    __syncthreads();
  }
  if (s_cnt < 3) { fail(); return; }
  if (threadIdx.x < 9) Rf[9 * pair + threadIdx.x] = static_cast<float>(s_R[threadIdx.x]);
  if (threadIdx.x < 3) tf[3 * pair + threadIdx.x] = static_cast<float>(s_t[threadIdx.x]);
  if (threadIdx.x == 0) n_inl[pair] = s_cnt;
}

// ================================================================================================
// ICP refinement of the Procrustes pose over the FULL depth clouds (pose_solver.py:289-315: Open3D registration_icp,
// point-to-point, max correspondence distance = PROCRUSTES.MAX_CORR_DIST, <= 30 iterations, relative fitness / rmse 1e-4).
// Both clouds are organised (one 3-D point per valid depth pixel), so the nearest neighbour of a transformed source point
// P inside the correspondence radius D is found EXACTLY by a window search around its projection into image 1: a target
// point within D of P lies within r = ceil(D (f + |u - c|) / (z - D)) + 1 pixels of it on each axis (the + 1 covers the
// rounding of the projection to a pixel and the float32 inverse of K). The window is clamped to kIcpMaxRadius; when the
// clamp cuts it, a point outside the clamped window is at least delta* = m z / (f + |u - c| + m), m = kIcpMaxRadius - 1,
// away from P (the same inequality solved for the distance), so the unclamped window is scanned only when no match
// closer than delta* was found. Source points with z <= D + 1 mm in camera 1 are not associated: exact as long as no
// target point is nearer than 2 D + 1 mm to camera 1. No k-d tree.
// State per pair (double[kIcpState]): [0..8] R, [9..11] t (current source -> target transform), [12] fitness, [13] rmse,
// [14] converged flag, [15] correspondences, [16] valid source points, [17] valid target points.
// Partial sums per pair and chunk of kIcpChunk source pixels (double[17]): n, sum p [3], sum q [3], sum p q^T [9],
// sum |p - q|^2 (p = transformed source point). The chunks depend on H W only, and icp_update_kernel adds them in chunk
// order, so a pair's result does not depend on the batch it runs in or on the GPU's SM count.
// ================================================================================================
__global__ void f32_to_f64_kernel(const float* __restrict__ a, double* __restrict__ b, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) b[i] = a[i];
}

constexpr int kIcpState = 18;
constexpr int kIcpMaxRadius = 96;
constexpr int kIcpChunk = 512;        // source pixels per association block (2 per thread)

__global__ void icp_count_kernel(const float* __restrict__ depth0, const float* __restrict__ depth1, int hw,
                                 const double* __restrict__ Rd, const double* __restrict__ td, double* __restrict__ state) {
  const int pair = blockIdx.y;
  __shared__ int s0[32], s1[32];
  int c0 = 0, c1 = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < hw; i += gridDim.x * blockDim.x) {
    c0 += depth0[static_cast<size_t>(pair) * hw + i] > 0.f;
    c1 += depth1[static_cast<size_t>(pair) * hw + i] > 0.f;
  }
  for (int o = 16; o > 0; o >>= 1) { c0 += __shfl_xor_sync(0xffffffffu, c0, o); c1 += __shfl_xor_sync(0xffffffffu, c1, o); }
  if ((threadIdx.x & 31) == 0) { s0[threadIdx.x >> 5] = c0; s1[threadIdx.x >> 5] = c1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0, b = 0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) { a += s0[w]; b += s1[w]; }
    atomicAdd(state + pair * kIcpState + 16, static_cast<double>(a));   // integer-valued: exact in any order
    atomicAdd(state + pair * kIcpState + 17, static_cast<double>(b));
    if (blockIdx.x == 0) {
      for (int k = 0; k < 9; ++k) state[pair * kIcpState + k] = Rd[9 * pair + k];
      for (int k = 0; k < 3; ++k) state[pair * kIcpState + 9 + k] = td[3 * pair + k];
    }
  }
}

// nearest target point to P with squared distance < best over pixels [u_lo, u_hi] x [v_lo, v_hi] of depth1 (row-major
// order, first on ties); z1 outside (zlo, zhi) (which also holds invalid depth 0) cannot be within D
__device__ __forceinline__ void icp_scan(const float* __restrict__ d1, int W, const float* Ki1, const double* P, float zlo,
                                         float zhi, int u_lo, int u_hi, int v_lo, int v_hi, double& best, double* Q) {
  for (int v = v_lo; v <= v_hi; ++v)
    for (int u = u_lo; u <= u_hi; ++u) {
      const float z1 = d1[v * W + u];
      if (!(z1 > zlo && z1 < zhi)) continue;
      double Y[3];
      backproject(Ki1, u, v, z1, Y);
      const double dx = Y[0] - P[0], dy = Y[1] - P[1], dz = Y[2] - P[2];
      const double dd = dx * dx + dy * dy + dz * dz;
      if (dd < best) { best = dd; Q[0] = Y[0]; Q[1] = Y[1]; Q[2] = Y[2]; }
    }
}

__global__ void __launch_bounds__(256) icp_assoc_kernel(const float* __restrict__ depth0, const float* __restrict__ depth1,
                                                        int H, int W, const float* __restrict__ K0s, const float* __restrict__ K1s,
                                                        float max_dist, const double* __restrict__ state,
                                                        double* __restrict__ partial) {
  const int pair = blockIdx.y;
  const double* st = state + pair * kIcpState;
  if (st[14] != 0.0 || !(st[0] == st[0])) return;                 // converged (or no initial pose): nothing to do
  __shared__ float s_Ki0[9], s_Ki1[9], s_K1[9];
  __shared__ double sh_red[8 * 17];
  if (threadIdx.x == 0) {
    inverse_K_f32(K0s + 9 * pair, s_Ki0);
    inverse_K_f32(K1s + 9 * pair, s_Ki1);
    for (int k = 0; k < 9; ++k) s_K1[k] = K1s[9 * pair + k];
  }
  __syncthreads();
  double R[9], t[3];
  for (int k = 0; k < 9; ++k) R[k] = st[k];
  for (int k = 0; k < 3; ++k) t[k] = st[9 + k];
  const float* d0 = depth0 + static_cast<size_t>(pair) * H * W;
  const float* d1 = depth1 + static_cast<size_t>(pair) * H * W;
  const double D = max_dist, D2 = D * D;
  const double fx = s_K1[0], fy = s_K1[4], cx = s_K1[2], cy = s_K1[5];
  const double rmax = static_cast<double>(W + H);                  // a radius that covers the whole image
  double a[17];
  for (int k = 0; k < 17; ++k) a[k] = 0.0;
  const int i_end = min(H * W, (blockIdx.x + 1) * kIcpChunk);
  for (int i = blockIdx.x * kIcpChunk + threadIdx.x; i < i_end; i += blockDim.x) {
    const float z0 = d0[i];
    if (!(z0 > 0.f)) continue;
    double X[3], P[3];
    backproject(s_Ki0, i % W, i / W, z0, X);
    mat3_vec(R, X, P);
    for (int k = 0; k < 3; ++k) P[k] += t[k];
    if (!(P[2] > D + 1e-3)) continue;                              // behind / too close to camera 1 (see above)
    const double up = fx * P[0] / P[2] + cx, vp = fy * P[1] / P[2] + cy;
    const double zr = 1.0 / (P[2] - D);
    const double au = fabs(up - cx), av = fabs(vp - cy);
    const double ru_full = fmin(rmax, ceil(D * (fx + au) * zr) + 1.0);
    const double rv_full = fmin(rmax, ceil(D * (fy + av) * zr) + 1.0);
    const int ru = min(kIcpMaxRadius, static_cast<int>(ru_full)), rv = min(kIcpMaxRadius, static_cast<int>(rv_full));
    // far outside the image the window is empty either way: clamp before the conversion to int
    const int uc = static_cast<int>(floor(fmin(fmax(up, -rmax - 2.0), W + rmax + 2.0) + 0.5));
    const int vc = static_cast<int>(floor(fmin(fmax(vp, -rmax - 2.0), H + rmax + 2.0) + 0.5));
    double best = D2, Q[3] = {0, 0, 0};
    // conservative float32 bounds of the depth band (P.z - D, P.z + D)
    const float zlo = __double2float_rd(P[2] - D), zhi = __double2float_ru(P[2] + D);
    icp_scan(d1, W, s_Ki1, P, zlo, zhi, max(0, uc - ru), min(W - 1, uc + ru), max(0, vc - rv), min(H - 1, vc + rv), best, Q);
    if (ru < ru_full || rv < rv_full) {
      constexpr double m = kIcpMaxRadius - 1;
      double dstar = D;
      if (ru < ru_full) dstar = fmin(dstar, m * P[2] / (fx + au + m));
      if (rv < rv_full) dstar = fmin(dstar, m * P[2] / (fy + av + m));
      dstar *= 1.0 - 1e-12;
      if (!(best < dstar * dstar)) {
        const int RU = static_cast<int>(ru_full), RV = static_cast<int>(rv_full);
        icp_scan(d1, W, s_Ki1, P, zlo, zhi, max(0, uc - RU), min(W - 1, uc + RU), max(0, vc - RV), min(H - 1, vc + RV),
                 best, Q);
      }
    }
    if (best < D2) {
      a[0] += 1.0;
      for (int r = 0; r < 3; ++r) {
        a[1 + r] += P[r]; a[4 + r] += Q[r];
        for (int c = 0; c < 3; ++c) a[7 + 3 * r + c] += P[r] * Q[c];
      }
      a[16] += best;
    }
  }
  block_sum_256<17>(a, sh_red);
  if (threadIdx.x == 0) {
    double* out = partial + (static_cast<size_t>(pair) * gridDim.x + blockIdx.x) * 17;
    for (int k = 0; k < 17; ++k) out[k] = a[k];
  }
}

// one warp per pair: the association's sums (chunk partials added in a fixed order), its fitness / rmse, the convergence
// test against the previous association (Open3D RegistrationICP: |d fitness| < rel_fitness and |d rmse| < rel_rmse),
// the Kabsch update composed onto the transform
__global__ void __launch_bounds__(64) icp_update_kernel(double* __restrict__ state, const double* __restrict__ partial,
                                                        int chunks, int P, int iter, double rel_fit, double rel_rmse) {
  const int pair = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (pair >= P) return;
  double* st = state + pair * kIcpState;
  if (st[14] != 0.0 || !(st[0] == st[0])) return;
  double a[17];
  for (int k = 0; k < 17; ++k) a[k] = 0.0;
  const double* pp = partial + static_cast<size_t>(pair) * chunks * 17;
  for (int c = lane; c < chunks; c += 32)
    for (int k = 0; k < 17; ++k) a[k] += pp[static_cast<size_t>(c) * 17 + k];
  for (int k = 0; k < 17; ++k)
    for (int o = 16; o > 0; o >>= 1) a[k] += __shfl_down_sync(0xffffffffu, a[k], o);
  if (lane != 0) return;
  const double n = a[0];
  const double fit = st[16] > 0.0 ? n / st[16] : 0.0, rmse = n > 0.0 ? sqrt(a[16] / n) : 0.0;
  const bool conv = iter > 0 && fabs(st[12] - fit) < rel_fit && fabs(st[13] - rmse) < rel_rmse;
  st[12] = fit; st[13] = rmse; st[15] = n;
  if (conv || n < 3.0) { st[14] = 1.0; }
  else {
    double Ru[9], tu[3];
    if (kabsch_from_sums(n, a + 1, a + 4, a + 7, Ru, tu)) {       // update maps the transformed source onto its correspondences
      double Rn[9], tn[3];
      mat3_mul(Ru, st, Rn);
      mat3_vec(Ru, st + 9, tn);
      for (int k = 0; k < 9; ++k) st[k] = Rn[k];
      for (int k = 0; k < 3; ++k) st[9 + k] = tn[k] + tu[k];
    } else {
      st[14] = 1.0;
    }
  }
}

__global__ void icp_finish_kernel(const double* __restrict__ state, int P, float* __restrict__ Rf, float* __restrict__ tf,
                                  int* __restrict__ n_inl) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= P) return;
  const double* st = state + pair * kIcpState;
  if (!(st[0] == st[0])) {                                         // NaN initial pose: the RANSAC stage failed, ICP does not run
    for (int k = 0; k < 9; ++k) Rf[9 * pair + k] = NAN;
    for (int k = 0; k < 3; ++k) tf[3 * pair + k] = NAN;
    n_inl[pair] = 0;
    return;
  }
  for (int k = 0; k < 9; ++k) Rf[9 * pair + k] = static_cast<float>(st[k]);
  for (int k = 0; k < 3; ++k) tf[3 * pair + k] = static_cast<float>(st[9 + k]);
  n_inl[pair] = static_cast<int>(st[12] * st[17]);                // pose_solver.py:319: int(fitness * len(pcl_1.points))
}

// ================================================================================================
// CONFIDENCE escalation (pose_solver._SolverBase on the device): after the round at `budget`, every pair still active
// records that budget (its outputs now hold that round's result) and stays active iff the stopping rule asks for more.
// Round 0 runs every pair (first_round); a pair with fewer correspondences than a minimal sample leaves with budget 0.
// ================================================================================================
__global__ void ransac_escalate_kernel(const int* __restrict__ offsets, const int* __restrict__ n_inl, int P, int max_pts,
                                       double confidence, int budget, int max_budget, int sample_size, int first_round,
                                       int* __restrict__ active, int* __restrict__ budgets) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= P || (!first_round && !active[pair])) return;
  const int N = min(offsets[pair + 1] - offsets[pair], max_pts);
  if (N < sample_size) {
    active[pair] = 0;
    budgets[pair] = 0;
    return;
  }
  budgets[pair] = budget;
  active[pair] = ransac_satisfied(confidence, n_inl[pair], N, budget, max_budget, sample_size) ? 0 : 1;
}

}  // namespace

// ================================================================================================
// host side
// ================================================================================================
struct PoseSolver {
  int max_pairs, max_pts, max_hyp;
  HypResult* results = nullptr;
  void* lo_out = nullptr;   // LoResult[max_pairs][kLoTopK]
  void* pts_norm = nullptr; // float4[max_pairs][max_pts]: normalised correspondences for the hypothesis kernel
  double *Rd = nullptr, *td = nullptr, *Xw = nullptr, *X1w = nullptr;
  float* uv = nullptr;
  int *vidx = nullptr, *nvalid = nullptr;
  int *active = nullptr, *budgets = nullptr;   // CONFIDENCE escalation: pair still solving / budget of its outputs
  unsigned int *dmin = nullptr, *dmin1 = nullptr;
  double* icp_state = nullptr;   // ICP refinement scratch (allocated on first use)
  double* icp_partial = nullptr; // ICP chunk partial sums [max_pairs][icp_chunks][17] (allocated / grown on use)
  int icp_chunks = 0;
  size_t total_pts;
};

int pose_solver_create(int max_pairs, int max_pts, int max_hyp, PoseSolver** out) {
  // correspondences of a pair live in shared memory in the LO / final / consensus kernels (16 B each): 8192 is the hard limit
  if (max_pairs < 1 || max_pts < 8 || max_pts > 8192 || max_hyp < kHypPerBlock) return MFR_ERR_ARG;
  auto* s = new PoseSolver();
  s->max_pairs = max_pairs; s->max_pts = max_pts; s->max_hyp = max_hyp;
  s->total_pts = static_cast<size_t>(max_pairs) * max_pts;
  const int blocks = (max_hyp + 31) / 32;   // the E-mat kernel may run with as few as 32 hypotheses per block
  bool ok = true;
  ok &= cudaMalloc(&s->results, sizeof(HypResult) * max_pairs * blocks) == cudaSuccess;
  ok &= cudaMalloc(&s->lo_out, sizeof(LoResult) * max_pairs * kLoTopK) == cudaSuccess;
  ok &= cudaMalloc(&s->pts_norm, sizeof(float4) * static_cast<size_t>(max_pairs) * s->max_pts) == cudaSuccess;
  ok &= cudaMalloc(&s->Rd, sizeof(double) * 9 * max_pairs) == cudaSuccess;
  ok &= cudaMalloc(&s->td, sizeof(double) * 3 * max_pairs) == cudaSuccess;
  ok &= cudaMalloc(&s->Xw, sizeof(double) * 3 * s->total_pts) == cudaSuccess;
  ok &= cudaMalloc(&s->X1w, sizeof(double) * 3 * s->total_pts) == cudaSuccess;
  ok &= cudaMalloc(&s->uv, sizeof(float) * 2 * s->total_pts) == cudaSuccess;
  ok &= cudaMalloc(&s->vidx, sizeof(int) * s->total_pts) == cudaSuccess;
  ok &= cudaMalloc(&s->nvalid, sizeof(int) * max_pairs) == cudaSuccess;
  ok &= cudaMalloc(&s->active, sizeof(int) * max_pairs) == cudaSuccess;
  ok &= cudaMalloc(&s->budgets, sizeof(int) * max_pairs) == cudaSuccess;
  ok &= cudaMalloc(&s->dmin, sizeof(unsigned int) * max_pairs) == cudaSuccess;
  ok &= cudaMalloc(&s->dmin1, sizeof(unsigned int) * max_pairs) == cudaSuccess;
  if (!ok) { pose_solver_destroy(s); return MFR_ERR_CUDA; }
  static bool attr_seen[64] = {};
  if (first_call_on_device(attr_seen)) {
    cudaFuncSetAttribute(emat_final_kernel<Scoring::kMsac>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16);
    cudaFuncSetAttribute(emat_lo_kernel<Scoring::kMsac>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16);
    cudaFuncSetAttribute(emat_final_kernel<Scoring::kMagsac>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16);
    cudaFuncSetAttribute(emat_lo_kernel<Scoring::kMagsac>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16);
    cudaFuncSetAttribute(scale_consensus_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 8);
    cudaFuncSetAttribute(pnp_hyp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 20);
    cudaFuncSetAttribute(procrustes_hyp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 24);
  }
  *out = s;
  return MFR_OK;
}

void pose_solver_destroy(PoseSolver* s) {
  if (!s) return;
  cudaFree(s->results); cudaFree(s->lo_out); cudaFree(s->pts_norm); cudaFree(s->Rd); cudaFree(s->td); cudaFree(s->Xw); cudaFree(s->uv);
  cudaFree(s->vidx); cudaFree(s->nvalid); cudaFree(s->active); cudaFree(s->budgets); cudaFree(s->dmin); cudaFree(s->dmin1); cudaFree(s->X1w); cudaFree(s->icp_state);
  cudaFree(s->icp_partial);
  delete s;
}

double* pose_solver_Rd(PoseSolver* s) { return s->Rd; }
double* pose_solver_td(PoseSolver* s) { return s->td; }

int pose_solver_debug_tensor(PoseSolver* s, const char* name, void** ptr, long long* words) {
  if (!s || !name || !ptr || !words) return MFR_ERR_ARG;
  const long long P = s->max_pairs, T = static_cast<long long>(s->total_pts);
  const long long blocks = (s->max_hyp + 31) / 32;
  const struct { const char* name; void* p; long long bytes; } bufs[] = {
      {"hyp_results", s->results, static_cast<long long>(sizeof(HypResult)) * P * blocks},
      {"lo_results", s->lo_out, static_cast<long long>(sizeof(LoResult)) * P * kLoTopK},
      {"pts_norm", s->pts_norm, 16 * T},
      {"Rd", s->Rd, 8 * 9 * P},
      {"td", s->td, 8 * 3 * P},
      {"Xw", s->Xw, 8 * 3 * T},
      {"uv", s->uv, 4 * 2 * T},
      {"vidx", s->vidx, 4 * T},
      {"nvalid", s->nvalid, 4 * P},
      {"dmin", s->dmin, 4 * P},
      {"X1w", s->X1w, 8 * 3 * T},
      {"dmin1", s->dmin1, 4 * P},
      {"icp_state", s->icp_state, 8 * kIcpState * P},
  };
  for (const auto& b : bufs)
    if (strcmp(b.name, name) == 0) {
      if (!b.p) return MFR_ERR_ARG;     // icp_state: no mfr_icp_refine call yet
      *ptr = b.p;
      *words = b.bytes / 4;
      return MFR_OK;
    }
  return MFR_ERR_ARG;
}

namespace {

// The hypothesis budgets of one solve: one entry for a fixed-budget call, h0, min(cap, 4 h0), ... up to the cap for an
// escalating one (at most 17 entries: the cap is an int).
struct BudgetSeq {
  int h[17];
  int n = 0;
  double confidence = 0.0;
  int cap = 0;
  int* budgets_out = nullptr;   // device int[P] or nullptr
};

BudgetSeq fixed_budget(const PoseSolver* s, int num_hyp) {
  BudgetSeq b;
  b.h[0] = b.cap = std::min(num_hyp, s->max_hyp);
  b.n = 1;
  return b;
}

int escalation_budgets(const PoseSolver* s, int num_hyp, double confidence, int max_hyp, int* budgets_out, BudgetSeq* b) {
  if (num_hyp < 1 || max_hyp < num_hyp || max_hyp > s->max_hyp) return MFR_ERR_ARG;
  b->h[0] = num_hyp;
  b->n = 1;
  if (confidence > 0.0)
    for (long long h = num_hyp; h < max_hyp;) {
      h = std::min<long long>(max_hyp, 4 * h);
      b->h[b->n++] = static_cast<int>(h);
    }
  b->confidence = confidence;
  b->cap = max_hyp;
  b->budgets_out = budgets_out;
  return MFR_OK;
}

// Runs round(h, active) for every budget h of `b`: round 0 on every pair (active = nullptr), each later round on the
// pairs the stopping rule kept active. All rounds are enqueued up front; no host synchronisation.
template <class Round>
int run_rounds(PoseSolver* s, const BudgetSeq& b, const int* offsets, int P, const int* n_inl, int sample_size,
               cudaStream_t st, Round round) {
  int* budgets = b.budgets_out ? b.budgets_out : s->budgets;
  for (int k = 0; k < b.n; ++k) {
    round(b.h[k], k == 0 ? nullptr : s->active);
    if (b.n > 1 || b.budgets_out)
      ransac_escalate_kernel<<<(P + 255) / 256, 256, 0, st>>>(offsets, n_inl, P, s->max_pts, b.confidence, b.h[k], b.cap,
                                                             sample_size, k == 0, s->active, budgets);
  }
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

}  // namespace

// kScore = kMagsac runs with lo_enabled = 1 (sigma-consensus++ from every LO candidate)
template <Scoring kScore>
static int emat_solve(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P, const float* K0,
                      const float* K1, float pix_thr, const BudgetSeq& b, unsigned long long seed, int lo_enabled,
                      float* R, float* t, int* n_inl, unsigned char* mask, cudaStream_t st) {
  if (P < 1 || P > s->max_pairs) return MFR_ERR_ARG;
  const size_t smem = static_cast<size_t>(s->max_pts) * 16;
  emat_normalise_kernel<<<dim3((s->max_pts + 255) / 256, P), 256, 0, st>>>(kpts0, kpts1, offsets, K0, K1, s->max_pts,
                                                                          static_cast<float4*>(s->pts_norm));
  // a round at budget h is the fixed-budget solve at h: the same hypotheses per block (so the same block partition
  // and LO candidates) and the same seed
  auto round = [&](int num_hyp, const int* active) {
    // hypotheses per block: 128 when that already gives >= 2 blocks per SM, else down to one warp per block
    // (enough pairs: full 128-thread blocks, one per SM beside the matcher's GEMM CTAs — see emat_hyp_kernel)
    int hpb = kHypPerBlock;
    while (hpb > 32 && static_cast<long long>(P) * ((num_hyp + hpb - 1) / hpb) < sm_count() / 2) hpb /= 2;
    const int blocks = (num_hyp + hpb - 1) / hpb;
    emat_hyp_kernel<kScore><<<dim3(blocks, P), hpb, 0, st>>>(static_cast<const float4*>(s->pts_norm), offsets, K0, K1, pix_thr,
                                                     num_hyp, seed, s->max_pts, s->results, active);
    emat_lo_kernel<kScore><<<dim3(P, kLoTopK), kLoThreads, smem, st>>>(kpts0, kpts1, offsets, K0, K1, pix_thr, blocks, s->max_pts,
                                                               s->results, static_cast<LoResult*>(s->lo_out), lo_enabled,
                                                               active);
    emat_final_kernel<kScore><<<P, kLoThreads, smem, st>>>(kpts0, kpts1, offsets, K0, K1, pix_thr, blocks, s->max_pts, s->results,
                                                   static_cast<const LoResult*>(s->lo_out), s->Rd, s->td, R, t, n_inl, mask,
                                                   lo_enabled, active);
  };
  return run_rounds(s, b, offsets, P, n_inl, 5, st, round);
}

int emat_ransac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                const float* K0, const float* K1, float pix_thr, int num_hyp, unsigned long long seed,
                int lo_enabled, float* R, float* t, int* n_inl, unsigned char* mask, cudaStream_t st) {
  if (num_hyp < 1) return MFR_ERR_ARG;
  return emat_solve<Scoring::kMsac>(s, kpts0, kpts1, offsets, P, K0, K1, pix_thr, fixed_budget(s, num_hyp), seed,
                                    lo_enabled, R, t, n_inl, mask, st);
}

int emat_ransac_escalate(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                         const float* K0, const float* K1, float pix_thr, int num_hyp, unsigned long long seed,
                         int lo_enabled, float* R, float* t, int* n_inl, unsigned char* mask, double confidence,
                         int max_hyp, int* budgets_out, cudaStream_t st) {
  BudgetSeq b;
  const int rc = escalation_budgets(s, num_hyp, confidence, max_hyp, budgets_out, &b);
  if (rc != MFR_OK) return rc;
  return emat_solve<Scoring::kMsac>(s, kpts0, kpts1, offsets, P, K0, K1, pix_thr, b, seed, lo_enabled, R, t, n_inl, mask,
                                    st);
}

int emat_magsac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P, const float* K0,
                const float* K1, float pix_thr, int num_hyp, unsigned long long seed, float* R, float* t, int* n_inl,
                unsigned char* mask, double confidence, int max_hyp, int* budgets_out, cudaStream_t st) {
  BudgetSeq b;
  const int rc = escalation_budgets(s, num_hyp, confidence, max_hyp, budgets_out, &b);
  if (rc != MFR_OK) return rc;
  return emat_solve<Scoring::kMagsac>(s, kpts0, kpts1, offsets, P, K0, K1, pix_thr, b, seed, 1, R, t, n_inl, mask, st);
}

int scale_from_depth(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                     const float* K0, const float* K1, const unsigned char* mask, const double* Rd,
                     const double* td, const float* depth0, const float* depth1, int H, int W,
                     float scale_thr, float* R_out, float* t_out, int* inliers, cudaStream_t st) {
  if (P < 1 || P > s->max_pairs) return MFR_ERR_ARG;
  const double* Rp = Rd ? Rd : s->Rd;
  const double* tp = td ? td : s->td;
  scale_consensus_kernel<<<P, 1024, static_cast<size_t>(s->max_pts) * 8, st>>>(
      kpts0, kpts1, offsets, K0, K1, mask, Rp, tp, depth0, depth1, H, W, static_cast<double>(scale_thr),
      s->max_pts, R_out, t_out, inliers);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

static int pnp_solve(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P, const float* K0,
                     const float* K1, const float* depth0, int H, int W, const BudgetSeq& b, float reproj_thr,
                     unsigned long long seed, float* R, float* t, int* n_inl, unsigned char* mask, cudaStream_t st) {
  if (P < 1 || P > s->max_pairs) return MFR_ERR_ARG;
  MFR_CUDA_CHECK(cudaMemsetAsync(s->dmin, 0x7f, sizeof(unsigned int) * P, st));
  depth_min_kernel<<<dim3(64, P), 256, 0, st>>>(depth0, static_cast<long long>(H) * W, s->dmin);
  pnp_prepare_kernel<<<P, 1024, 0, st>>>(kpts0, kpts1, offsets, K0, depth0, H, W, s->dmin, s->max_pts, s->Xw,
                                         s->uv, s->vidx, s->nvalid);
  auto round = [&](int num_hyp, const int* active) {
    const int blocks = (num_hyp + kHypPerBlock - 1) / kHypPerBlock;
    pnp_hyp_kernel<<<dim3(blocks, P), kHypPerBlock, static_cast<size_t>(s->max_pts) * 20, st>>>(
        s->Xw, s->uv, offsets, s->nvalid, K1, reproj_thr, num_hyp, seed, s->max_pts, s->results, active);
    pnp_final_kernel<<<P, 256, 0, st>>>(s->Xw, s->uv, s->vidx, offsets, s->nvalid, K1, reproj_thr, blocks,
                                        s->max_pts, s->results, R, t, n_inl, mask, active);
  };
  return run_rounds(s, b, offsets, P, n_inl, 4, st, round);
}

int pnp_ransac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
               const float* K0, const float* K1, const float* depth0, int H, int W, int num_hyp,
               float reproj_thr, unsigned long long seed, float* R, float* t, int* n_inl,
               unsigned char* mask, cudaStream_t st) {
  if (num_hyp < 1) return MFR_ERR_ARG;
  return pnp_solve(s, kpts0, kpts1, offsets, P, K0, K1, depth0, H, W, fixed_budget(s, num_hyp), reproj_thr, seed, R, t,
                   n_inl, mask, st);
}

int pnp_ransac_escalate(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                        const float* K0, const float* K1, const float* depth0, int H, int W, int num_hyp,
                        float reproj_thr, unsigned long long seed, float* R, float* t, int* n_inl,
                        unsigned char* mask, double confidence, int max_hyp, int* budgets_out, cudaStream_t st) {
  BudgetSeq b;
  const int rc = escalation_budgets(s, num_hyp, confidence, max_hyp, budgets_out, &b);
  if (rc != MFR_OK) return rc;
  return pnp_solve(s, kpts0, kpts1, offsets, P, K0, K1, depth0, H, W, b, reproj_thr, seed, R, t, n_inl, mask, st);
}

int procrustes_ransac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                      const float* K0, const float* K1, const float* depth0, const float* depth1, int H, int W,
                      int num_hyp, float max_corr_dist, unsigned long long seed, float* R, float* t, int* n_inl,
                      cudaStream_t st) {
  if (P < 1 || P > s->max_pairs || num_hyp < 1) return MFR_ERR_ARG;
  num_hyp = std::min(num_hyp, s->max_hyp);
  const int blocks = (num_hyp + kHypPerBlock - 1) / kHypPerBlock;
  MFR_CUDA_CHECK(cudaMemsetAsync(s->dmin, 0x7f, sizeof(unsigned int) * P, st));
  MFR_CUDA_CHECK(cudaMemsetAsync(s->dmin1, 0x7f, sizeof(unsigned int) * P, st));
  depth_min_kernel<<<dim3(64, P), 256, 0, st>>>(depth0, static_cast<long long>(H) * W, s->dmin);
  depth_min_kernel<<<dim3(64, P), 256, 0, st>>>(depth1, static_cast<long long>(H) * W, s->dmin1);
  procrustes_prepare_kernel<<<P, 1024, 0, st>>>(kpts0, kpts1, offsets, K0, K1, depth0, depth1, H, W, s->dmin,
                                                s->dmin1, s->max_pts, s->Xw, s->X1w, s->nvalid);
  procrustes_hyp_kernel<<<dim3(blocks, P), kHypPerBlock, static_cast<size_t>(s->max_pts) * 24, st>>>(
      s->Xw, s->X1w, offsets, s->nvalid, max_corr_dist, num_hyp, seed, s->max_pts, s->results);
  procrustes_final_kernel<<<P, 256, 0, st>>>(s->Xw, s->X1w, offsets, s->nvalid, max_corr_dist, blocks, s->max_pts, s->results, R,
                                             t, n_inl);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int icp_refine(PoseSolver* s, const float* depth0, const float* depth1, int H, int W, int P, const float* K0, const float* K1,
               const float* R_in, const float* t_in, float max_corr_dist, int max_iter, float rel_fitness, float rel_rmse,
               float* R, float* t, int* n_inl, cudaStream_t st) {
  if (P < 1 || P > s->max_pairs || max_iter < 1 || H < 1 || W < 1) return MFR_ERR_ARG;
  const int chunks = static_cast<int>((static_cast<long long>(H) * W + kIcpChunk - 1) / kIcpChunk);
  if (!s->icp_state) {
    if (cudaMalloc(&s->icp_state, sizeof(double) * (kIcpState + 12) * s->max_pairs) != cudaSuccess) return MFR_ERR_CUDA;
  }
  if (chunks > s->icp_chunks) {     // first call at a larger frame (not inside a graph capture: warm up at that size first)
    cudaFree(s->icp_partial);
    s->icp_partial = nullptr;
    s->icp_chunks = 0;
    if (cudaMalloc(&s->icp_partial, sizeof(double) * 17 * chunks * s->max_pairs) != cudaSuccess) return MFR_ERR_CUDA;
    s->icp_chunks = chunks;
  }
  double* state = s->icp_state;
  double* Rd = state + static_cast<size_t>(kIcpState) * s->max_pairs;      // initial pose in double: R [P][9] then t [P][3]
  double* td = Rd + static_cast<size_t>(9) * s->max_pairs;
  MFR_CUDA_CHECK(cudaMemsetAsync(state, 0, sizeof(double) * kIcpState * s->max_pairs, st));
  f32_to_f64_kernel<<<(9 * P + 255) / 256, 256, 0, st>>>(R_in, Rd, 9 * P);
  f32_to_f64_kernel<<<(3 * P + 255) / 256, 256, 0, st>>>(t_in, td, 3 * P);
  icp_count_kernel<<<dim3(64, P), 256, 0, st>>>(depth0, depth1, H * W, Rd, td, state);
  for (int it = 0; it <= max_iter; ++it) {
    // association under the current transform; the update kernel evaluates it (fitness, rmse), tests convergence against the
    // previous association and applies the Kabsch step. The last pass (it == max_iter) only evaluates.
    icp_assoc_kernel<<<dim3(chunks, P), 256, 0, st>>>(depth0, depth1, H, W, K0, K1, max_corr_dist, state, s->icp_partial);
    icp_update_kernel<<<(P + 1) / 2, 64, 0, st>>>(state, s->icp_partial, chunks, P, it, it == max_iter ? 1e300 : rel_fitness,
                                                 it == max_iter ? 1e300 : rel_rmse);
  }
  icp_finish_kernel<<<(P + 63) / 64, 64, 0, st>>>(state, P, R, t, n_inl);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

}  // namespace mfr
