// Fused SuperGlue softmax attention (bf16 engine mode) on wgmma. See sg_attention.cuh for the op.
//
// One CTA per (query tile of 128 rows, head, image), three warpgroups:
//   * warpgroup 0: the TMA producer (warp 0; the warpgroup hands its registers to the consumers with setmaxnreg). It
//     loads the query tile once, then streams the partner image's key and value tiles (128 keys x 64 channels each,
//     128B-swizzled) through a ring of kStages slots, with a full and an empty mbarrier per slot. Only the tiles that
//     hold keys below the partner's count are loaded; rows past max_kp arrive zero-filled.
//   * warpgroups 1 and 2: the consumers, query rows 0-63 and 64-127 of the tile. Per key tile:
//       - S [64 x 128] = Q K^T (wgmma, both operands K-major in shared memory), fp32 in registers;
//       - keys at or past the count are set to -inf (last tile only), the running row max and row sum are updated
//         (online softmax, fp32; exp2 of the scores scaled by log2(e) / 8), and the output is rescaled;
//       - P is rounded to bf16 in registers, where the S fragment already has the layout of a wgmma A fragment, and
//         O [64 x 64] += P V runs with A from registers and V as an N-major B operand (imm-trans-b), so V needs no
//         transpose;
//       - once that group has completed, each warp hands the slot back.
//     The epilogue divides by the row sum and writes bf16 messages; rows at or past the query count are written as 0.
// Every reduction has a fixed order (keys in tile order, a fixed shuffle tree across the four lanes of a quad), so a
// row's message depends only on its own image pair.
#include "sg_attention.cuh"
#include "wgmma.cuh"

#include <cstring>
#include <mutex>

namespace mfr {

namespace {

constexpr int kQT = 128;                  // query rows per CTA: 64 per consumer warpgroup
constexpr int kKT = 128;                  // keys per K / V tile
constexpr int kStages = 4;                // K / V ring depth
constexpr int kThreads = 384;             // producer warpgroup + two consumer warpgroups
constexpr int kConsumerWarps = 8;
constexpr uint32_t kTile = 128 * 128;     // 128 rows x 64 bf16 channels (16 KB)
constexpr int kSmem = static_cast<int>((1 + 2 * kStages) * kTile) + 1024;
constexpr uint64_t kDescHi = (1ull << 16) | (64ull << 32) | (1ull << 62);   // 128B swizzle, 1 KB between 8-row groups
__device__ __forceinline__ uint64_t desc(uint32_t a) { return kDescHi | ((a >> 4) & 0x3fffu); }

__device__ __forceinline__ uint32_t bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

__global__ void __launch_bounds__(kThreads, 1) sg_attention_kernel(const __grid_constant__ SgAttentionParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_bar[1 + 2 * kStages];
  const int img = blockIdx.z, head = blockIdx.y, q0 = blockIdx.x * kQT;
  const int src = img ^ p.cross;
  const int nq = min(max(p.counts[img], 0), p.max_kp), nk = min(max(p.counts[src], 0), p.max_kp);
  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  unsigned short* out = p.msg + (static_cast<long long>(img) * p.max_kp + q0) * p.ldo + 64 * head;
  const int rows = min(kQT, p.max_kp - q0);   // rows of this image in the tile

  if (q0 >= nq || nk == 0) {   // no live query row, or nothing to attend to: zero messages
    for (int i = tid; i < rows * 32; i += kThreads)
      reinterpret_cast<uint32_t*>(out + static_cast<long long>(i >> 5) * p.ldo)[i & 31] = 0u;
    return;
  }
  const int n_kt = (nk + kKT - 1) / kKT;

  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = base;
  auto sK = [&](int s) { return base + (1 + 2 * s) * kTile; };
  auto sV = [&](int s) { return base + (2 + 2 * s) * kTile; };
  const uint32_t q_full = smem_u32(&s_bar[0]);
  auto full = [&](int s) { return smem_u32(&s_bar[1 + s]); };
  auto empty = [&](int s) { return smem_u32(&s_bar[1 + kStages + s]); };

  if (tid == 0) {
    tma_prefetch_desc(&p.tm);
    mbar_init(q_full, 1);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (warp 0)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0) {
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(q_full, kTile);
        tma_load_3d(sQ, &p.tm, q_full, 64 * head, q0, img);
      }
      for (int t = 0; t < n_kt; ++t) {
        const int s = t % kStages;
        wait_bounded(empty(s), static_cast<uint32_t>(((t / kStages) & 1) ^ 1));
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(full(s), 2 * kTile);
          tma_load_3d(sK(s), &p.tm, full(s), 256 + 64 * head, t * kKT, src);
          tma_load_3d(sV(s), &p.tm, full(s), 512 + 64 * head, t * kKT, src);
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers (warpgroups 1 and 2)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = (warp >> 2) - 1;                    // query rows 64 wg .. 64 wg + 63 of the tile
  const uint32_t aQ = sQ + wg * 64 * 128;
  const int cq = 2 * (lane & 3);                     // fragment columns 8j + cq, 8j + cq + 1
  constexpr float kScale = 0.125f * 1.4426950408889634f;   // 1 / sqrt(64), in base 2
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: this lane's share of the row sum

  wait_bounded(q_full, 0);
  for (int t = 0; t < n_kt; ++t) {
    const int s = t % kStages;
    wait_bounded(full(s), static_cast<uint32_t>((t / kStages) & 1));
    float sc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sc[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_bf16<128>(sc, desc(aQ) + 2 * k, desc(sK(s)) + 2 * k);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);

    if ((t + 1) * kKT > nk) {   // the last tile: keys at or past the count get zero weight
      const int lim = nk - t * kKT;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * j + cq + e >= lim) { sc[4 * j + e] = -INFINITY; sc[4 * j + 2 + e] = -INFINITY; }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = m_run[h];
#pragma unroll
      for (int j = 0; j < 16; ++j) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * h], sc[4 * j + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      // every tile has a live key, so mx is finite; on the first tile m_run is -inf and corr 0
      const float corr = exp2f((m_run[h] - mx) * kScale);
      const float mc = mx * kScale;
      m_run[h] = mx;
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float pv = exp2f(fmaf(sc[4 * j + 2 * h + e], kScale, -mc));
          sc[4 * j + 2 * h + e] = pv;
          sum += pv;
        }
      l_run[h] = l_run[h] * corr + sum;
#pragma unroll
      for (int j = 0; j < 8; ++j) { o[4 * j + 2 * h] *= corr; o[4 * j + 2 * h + 1] *= corr; }
    }
    // P as bf16 A fragments: keys 16 u .. 16 u + 15 are the S fragment's column groups 2u and 2u + 1
    uint32_t pa[8][4];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      pa[u][0] = bf16x2(sc[8 * u + 0], sc[8 * u + 1]);
      pa[u][1] = bf16x2(sc[8 * u + 2], sc[8 * u + 3]);
      pa[u][2] = bf16x2(sc[8 * u + 4], sc[8 * u + 5]);
      pa[u][3] = bf16x2(sc[8 * u + 6], sc[8 * u + 7]);
    }
    wgmma_fence();
#pragma unroll
    for (int u = 0; u < 8; ++u) wgmma_bf16_n64_rs(o, pa[u], desc(sV(s)) + u * (2048 >> 4));   // 16 keys = 2 KB
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(empty(s));
  }

  // ---- epilogue: O / row sum -> bf16 messages, zero rows past the query count
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;   // >= 1: the row max contributes exp2(0)
    const int r = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    if (r < rows) {
      const bool live = q0 + r < nq;
      uint32_t* orow = reinterpret_cast<uint32_t*>(out + static_cast<long long>(r) * p.ldo + cq);
#pragma unroll
      for (int j = 0; j < 8; ++j) orow[4 * j] = live ? bf16x2(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv) : 0u;
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(f);
  });
  return fn;
}

}  // namespace

int sg_attention_build(const void* qkv, long long ldq, const int* counts, int n_img, int max_kp, int cross, void* msg,
                       long long ldo, SgAttentionParams* p) {
  if (n_img < 1 || n_img > 65535 || max_kp < 16 || max_kp > 2048 || (max_kp % 16) || (cross != 0 && cross != 1) ||
      (cross && (n_img & 1)))
    return MFR_ERR_ARG;
  if (!qkv || !counts || !msg || ldq < 768 || (ldq % 8) || (reinterpret_cast<uintptr_t>(qkv) & 15) || ldo < 256 ||
      (ldo & 1) || (reinterpret_cast<uintptr_t>(msg) & 3))
    return MFR_ERR_ARG;
  EncodeTiledFn enc = encode_fn();
  if (!enc) return MFR_ERR_CUDA;
  memset(p, 0, sizeof(*p));
  cuuint64_t dims[3] = {768, static_cast<cuuint64_t>(max_kp), static_cast<cuuint64_t>(n_img)};
  cuuint64_t strides[2] = {static_cast<cuuint64_t>(ldq) * 2, static_cast<cuuint64_t>(ldq) * 2 * max_kp};
  cuuint32_t box[3] = {64, static_cast<cuuint32_t>(kKT), 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&p->tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(qkv), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[mfr_b200] sg_attention: cuTensorMapEncodeTiled failed: %d\n", static_cast<int>(r));
    return MFR_ERR_CUDA;
  }
  p->counts = counts;
  p->msg = static_cast<unsigned short*>(msg);
  p->ldo = ldo;
  p->n_img = n_img; p->max_kp = max_kp; p->cross = cross;
  return MFR_OK;
}

int sg_attention_launch(const SgAttentionParams& p, cudaStream_t st) {
  static bool attr_seen[64] = {};
  if (first_call_on_device(attr_seen))
    MFR_CUDA_CHECK(cudaFuncSetAttribute(sg_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  sg_attention_kernel<<<dim3((p.max_kp + kQT - 1) / kQT, 4, p.n_img), kThreads, kSmem, st>>>(p);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

}  // namespace mfr
