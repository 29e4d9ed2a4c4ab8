// Fused LoFTREncoderLayer tail (bf16 engine mode) on wgmma. See encoder_tail.cuh for the op.
//
// Persistent, one CTA per SM, 128-row tiles of token rows, three warpgroups:
//   * warpgroup 0: the TMA producer (warp 0; the warpgroup hands its registers to the consumers with setmaxnreg). Per
//     row tile, in the order the consumers use them, it loads A2 = [x | message] (the x half of the bf16 token shadow
//     and the message, 128 rows, 128B-swizzled k-blocks of 64 columns), prefetches the tile's fp32 x rows into L2 for
//     the LayerNorm2 epilogue, then loads every weight tile of the chain ([<= 128 output rows x 64 input columns]) into
//     a ring of slots, as deep as shared memory allows, with a full and an empty mbarrier per slot.
//   * warpgroups 1 and 2: the consumers, rows 0-63 and 64-127 of the tile. Both read every weight tile from the same
//     slot, so the weights cross L2 once per 128 rows. Per tile and warpgroup:
//       - merge: D1 [64 x C] = message * Wm^T in registers (C / 128 accumulators of m64n128); LayerNorm1 on the fragments
//         (row statistics across the four lanes of a quad), written as bf16 over the message half of A2: A2 is now the
//         mlp.0 operand [x | norm1(merge(message))].
//       - the 2C-wide hidden layer in chunks (64 columns at C = 256, 128 at C = 128): D2 = A2 * W0[chunk]^T (registers),
//         relu, bf16 into the warpgroup's rows of the swizzled operand buffer H, then D3 [64 x C] += H * W2[:, chunk]^T
//         (registers). 2C-wide rows never exist anywhere.
//       - LayerNorm2 on D3, x += it (fp32), the bf16 shadow rewritten from the new x.
//     A consumer never issues a load. Each warp hands a weight slot back (an arrive on its empty barrier) once the wgmma
//     group that read it has completed, and A2 once the last mlp.0 chunk has read it, so the next tile's A2 arrives
//     while the last mlp.2 tiles and the LayerNorm2 epilogue run.
// HBM traffic per row: the message and x shadow read, x read and written, the shadow written; every intermediate stays
// on the SM.
#include "encoder_tail.cuh"
#include "wgmma.cuh"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <mutex>

namespace mfr {

int conv_gemm_num_sms();

namespace {

constexpr int kRows = 128;                // token rows per tile: 64 per warpgroup (the M of its wgmma)
constexpr int kThreads = 384;             // producer warpgroup + two consumer warpgroups
constexpr int kConsumerWarps = 8;
constexpr uint32_t kKb = kRows * 128;     // one 128-row x 64-column bf16 operand k-block (16 KB)
constexpr uint32_t kWgKb = 64 * 128;      // warpgroup w's 64 rows of a k-block start at w * kWgKb
constexpr uint32_t kWTile = 128 * 128;    // one weight slot: 128 output rows x 64 input columns (16 KB)
constexpr uint64_t kDescHi = (1ull << 16) | (64ull << 32) | (1ull << 62);   // K-major, 128B swizzle, 1024 B atoms
__device__ __forceinline__ uint64_t desc(uint32_t a) { return kDescHi | ((a >> 4) & 0x3fffu); }

template <int C>
struct Cfg {
  static constexpr int KB1 = C / 64;                 // k-blocks of C columns
  static constexpr int NH = C / 128;                 // 128-column accumulators of a C-wide result
  // hidden-layer chunk width: 64 columns at C = 256 (the merge / mlp.2 accumulators already take 128 registers),
  // 128 at C = 128
  static constexpr int QW = C == 256 ? 64 : 128;
  static constexpr int QK = QW / 64;                 // k-blocks of one hidden chunk
  static constexpr int NQ = 2 * C / QW;              // chunks of the hidden layer
  static constexpr int T_MERGE = NH * KB1;           // weight tiles of the merge GEMM
  static constexpr int T_CHUNK = 2 * KB1 + NH * QK;  // weight tiles of one hidden chunk: mlp.0 (K = 2C), mlp.2 (K = QW)
  static constexpr int T_ROW = T_MERGE + NQ * T_CHUNK;
  static constexpr uint32_t A2 = 2 * KB1 * kKb;
  static constexpr uint32_t H = QK * kKb;
  // weight slots: what shared memory holds next to A2 and H (224 KB in all at both widths). The per-tile traffic needs
  // depth to hide the L2 latency.
  static constexpr int WS = C == 256 ? 5 : 8;
  static constexpr int SMEM = static_cast<int>(A2 + H + WS * kWTile) + 1024;
};

// weight tile t (0 <= t < T_ROW) of a row tile's sequence: tensor map, (input column, output row) coordinates, bytes
template <int C>
__device__ __forceinline__ uint32_t wtile(const EncoderTailParams& p, int t, const CUtensorMap*& tm, int& k0, int& n0) {
  using G = Cfg<C>;
  if (t < G::T_MERGE) {
    tm = &p.tmWm; n0 = (t / G::KB1) * 128; k0 = (t % G::KB1) * 64;
    return kWTile;
  }
  t -= G::T_MERGE;
  const int q = t / G::T_CHUNK;
  int u = t - q * G::T_CHUNK;
  if (u < 2 * G::KB1) {
    tm = &p.tmW0; n0 = q * G::QW; k0 = u * 64;
    return G::QW * 128;
  }
  u -= 2 * G::KB1;
  tm = &p.tmW2; n0 = (u / G::QK) * 128; k0 = q * G::QW + (u % G::QK) * 64;
  return kWTile;
}

__device__ __forceinline__ uint32_t bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// mean and 1 / std (LayerNorm, eps 1e-5) of fragment row h: the row's C values sit in the four lanes of a quad
template <int NH>
__device__ __forceinline__ void row_stats(const float (&a)[NH][64], int h, float& mean, float& rstd) {
  constexpr float kInvC = 1.f / (NH * 128);
  float s = 0.f;
#pragma unroll
  for (int nh = 0; nh < NH; ++nh)
#pragma unroll
    for (int j = 0; j < 16; ++j) s += a[nh][4 * j + 2 * h] + a[nh][4 * j + 2 * h + 1];
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  mean = s * kInvC;
  float q = 0.f;
#pragma unroll
  for (int nh = 0; nh < NH; ++nh)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float d0 = a[nh][4 * j + 2 * h] - mean, d1 = a[nh][4 * j + 2 * h + 1] - mean;
      q += d0 * d0 + d1 * d1;
    }
  q += __shfl_xor_sync(0xffffffffu, q, 1);
  q += __shfl_xor_sync(0xffffffffu, q, 2);
  rstd = 1.f / sqrtf(q * kInvC + 1e-5f);
}

// v, hidden from the optimiser: values derived from it are recomputed where it is taken instead of hoisted out of loops
__device__ __forceinline__ int opaque(int v) {
  asm volatile("mov.b32 %0, %0;" : "+r"(v));
  return v;
}
__device__ __forceinline__ const float* opaque(const float* v) {
  asm volatile("mov.b64 %0, %0;" : "+l"(v));
  return v;
}

__device__ __forceinline__ void prefetch_l2(const void* ptr, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(ptr), "r"(bytes) : "memory");
}

template <int C>
__global__ void __launch_bounds__(kThreads, 1) encoder_tail_kernel(const __grid_constant__ EncoderTailParams p) {
  using G = Cfg<C>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_bar[2 + 2 * G::WS];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sA = base, sH = base + G::A2, sW = sH + G::H;
  const uint32_t a_full = smem_u32(&s_bar[0]), a_empty = smem_u32(&s_bar[1]);
  auto w_full = [&](int s) { return smem_u32(&s_bar[2 + s]); };
  auto w_empty = [&](int s) { return smem_u32(&s_bar[2 + G::WS + s]); };
  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;

  long long live = p.rows_cap;
  if (p.dyn_rows != nullptr) live = max(0LL, min(live, static_cast<long long>(*p.dyn_rows)));
  const int tiles_img = static_cast<int>((live + kRows - 1) / kRows);
  const int n_tiles = tiles_img * p.n_img;
  const int my_tiles = static_cast<int>(blockIdx.x) < n_tiles ? (n_tiles - 1 - static_cast<int>(blockIdx.x)) / gridDim.x + 1 : 0;
  if (my_tiles == 0) return;

  if (tid == 0) {
    tma_prefetch_desc(&p.tmMsg); tma_prefetch_desc(&p.tmX);
    tma_prefetch_desc(&p.tmWm); tma_prefetch_desc(&p.tmW0); tma_prefetch_desc(&p.tmW2);
    mbar_init(a_full, 1);
    mbar_init(a_empty, kConsumerWarps);
    for (int s = 0; s < G::WS; ++s) {
      mbar_init(w_full(s), 1);
      mbar_init(w_empty(s), kConsumerWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer (warp 0)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0) {
      long long gi = 0;   // weight tiles issued
      uint32_t a_ph = 1;  // a fresh barrier's preceding phase counts as complete
      for (int it = 0; it < my_tiles; ++it) {
        const int item = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x);
        const int img = item / tiles_img, tt = item - img * tiles_img;
        const int r0 = static_cast<int>(img * p.rows_cap) + tt * kRows;
        wait_bounded(a_empty, a_ph);
        a_ph ^= 1u;
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(a_full, G::A2);
          for (int kb = 0; kb < G::KB1; ++kb) {
            tma_load_2d(sA + kb * kKb, &p.tmX, a_full, kb * 64, r0);
            tma_load_2d(sA + (G::KB1 + kb) * kKb, &p.tmMsg, a_full, kb * 64, r0);
          }
        }
        // the tile's live fp32 x rows into L2 for the LayerNorm2 epilogue, widened to 16-byte bounds (bulk prefetch
        // granularity)
        const int n_live = static_cast<int>(min(static_cast<long long>(kRows), live - static_cast<long long>(tt) * kRows));
        for (int r = lane; r < n_live; r += 32) {
          const uintptr_t a = reinterpret_cast<uintptr_t>(p.x + (r0 + r) * p.ldx);
          const uintptr_t a0 = a & ~uintptr_t(15), a1 = (a + C * sizeof(float) + 15) & ~uintptr_t(15);
          prefetch_l2(reinterpret_cast<const void*>(a0), static_cast<uint32_t>(a1 - a0));
        }
        for (int t = 0; t < G::T_ROW; ++t, ++gi) {
          const int s = static_cast<int>(gi % G::WS);
          wait_bounded(w_empty(s), static_cast<uint32_t>(((gi / G::WS) & 1) ^ 1));
          if (elect_one_sync()) {
            const CUtensorMap* tm;
            int k0, n0;
            const uint32_t bytes = wtile<C>(p, t, tm, k0, n0);
            mbar_arrive_expect_tx(w_full(s), bytes);
            tma_load_2d(sW + s * kWTile, tm, w_full(s), k0, n0);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers (warpgroups 1 and 2)
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  const int wg = (warp >> 2) - 1;                           // rows 64 wg .. 64 wg + 63 of each tile
  const uint32_t sAw = sA + wg * kWgKb, sHw = sH + wg * kWgKb;
  auto wg_sync = [&]() { named_bar_sync(1 + wg, 128); };
  auto arrive = [&](uint32_t bar) {
    __syncwarp();
    if (lane == 0) mbar_arrive(bar);
  };
  long long g = 0, held = -1;   // weight tiles consumed; the tile read by the wgmma group still in flight (-1: none)
  auto release = [&]() {        // the group in flight has completed: its slot goes back to the producer
    if (held >= 0) arrive(w_empty(static_cast<int>(held % G::WS)));
    held = -1;
  };
  // one weight tile: 4 k-steps of (A k-block at a_addr) x (tile)^T into d; then the previous tile's group has completed
  auto step = [&](auto& d, uint32_t a_addr) {
    constexpr int N = 2 * static_cast<int>(sizeof(d) / sizeof(float));
    const int s = static_cast<int>(g % G::WS);
    wait_bounded(w_full(s), static_cast<uint32_t>((g / G::WS) & 1));
    const uint32_t b_addr = sW + s * kWTile;
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_bf16<N>(d, desc(a_addr) + 2 * k, desc(b_addr) + 2 * k);
    wgmma_commit();
    wgmma_wait<1>();
    release();
    held = g++;
  };

  const int rq0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
  const int cq0 = 2 * (lane & 3);
  uint32_t a_ph = 0;
  for (int it = 0; it < my_tiles; ++it) {
    const int item = static_cast<int>(blockIdx.x) + it * static_cast<int>(gridDim.x);
    const int img = item / tiles_img, tt = item - img * tiles_img;
    // tile rows rq and rq + 8 of the fragments, fragment columns 8j + cq, 8j + cq + 1, and the LayerNorm parameters.
    // Taken per tile: the shared memory addresses and parameter loads derived from them are tile-invariant, and hoisted
    // out of the loop they hold ~100 (addresses) and C (parameters) registers for the kernel's lifetime.
    const int rq = opaque(rq0), cq = opaque(cq0);
    const float *g1 = opaque(p.g1), *b1 = opaque(p.b1), *g2 = opaque(p.g2), *b2 = opaque(p.b2);
    wait_bounded(a_full, a_ph);
    a_ph ^= 1u;

    // ---- merge + LayerNorm1 -> message half of A2 (bf16)
    float acc[G::NH][64];
#pragma unroll
    for (int nh = 0; nh < G::NH; ++nh)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[nh][i] = 0.f;
#pragma unroll
    for (int nh = 0; nh < G::NH; ++nh)
      for (int kb = 0; kb < G::KB1; ++kb) step(acc[nh], sAw + (G::KB1 + kb) * kKb);
    wgmma_wait<0>();
    release();
#pragma unroll
    for (int nh = 0; nh < G::NH; ++nh) wgmma_fence_regs(acc[nh]);
    wg_sync();   // every warp's merge MMAs have read the message before it is overwritten
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mean, rstd;
      row_stats<G::NH>(acc, h, mean, rstd);
#pragma unroll
      for (int nh = 0; nh < G::NH; ++nh)
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = nh * 128 + 8 * j + cq;
          const float y0 = (acc[nh][4 * j + 2 * h] - mean) * rstd * __ldg(g1 + col) + __ldg(b1 + col);
          const float y1 = (acc[nh][4 * j + 2 * h + 1] - mean) * rstd * __ldg(g1 + col + 1) + __ldg(b1 + col + 1);
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(sw_addr(sA, rq + 8 * h, C + col, kKb)), "r"(bf16x2(y0, y1)) : "memory");
        }
    }
    fence_proxy_async_smem();
    wg_sync();

    // ---- hidden layer in chunks: mlp.0 + relu -> H (bf16), mlp.2 accumulates into acc3
    float acc3[G::NH][64];
#pragma unroll
    for (int nh = 0; nh < G::NH; ++nh)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc3[nh][i] = 0.f;
    for (int q = 0; q < G::NQ; ++q) {
      float acc2[G::QW / 2];
#pragma unroll
      for (int i = 0; i < G::QW / 2; ++i) acc2[i] = 0.f;
      for (int kb = 0; kb < 2 * G::KB1; ++kb) step(acc2, sAw + kb * kKb);
      wgmma_wait<0>();   // this chunk's mlp.0 and the previous chunk's mlp.2 (reads of H) have completed
      release();
      wgmma_fence_regs(acc2);
      if (q == G::NQ - 1) arrive(a_empty);   // A2 is free for the next row tile
      wg_sync();
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < G::QW / 8; ++j) {
          const float y0 = fmaxf(acc2[4 * j + 2 * h], 0.f), y1 = fmaxf(acc2[4 * j + 2 * h + 1], 0.f);
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(sw_addr(sH, rq + 8 * h, 8 * j + cq, kKb)), "r"(bf16x2(y0, y1)) : "memory");
        }
      fence_proxy_async_smem();
      wg_sync();
#pragma unroll
      for (int nh = 0; nh < G::NH; ++nh)
        for (int kb = 0; kb < G::QK; ++kb) step(acc3[nh], sHw + kb * kKb);
    }
    wgmma_wait<0>();
    release();
#pragma unroll
    for (int nh = 0; nh < G::NH; ++nh) wgmma_fence_regs(acc3[nh]);

    // ---- LayerNorm2 + residual: x (fp32) and its bf16 shadow, live rows only
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mean, rstd;
      row_stats<G::NH>(acc3, h, mean, rstd);
      const int r = tt * kRows + rq + 8 * h;
      if (r < live) {
        const long long grow = img * p.rows_cap + r;
        float* xr = p.x + grow * p.ldx;
        unsigned short* xbr = p.xb + grow * p.ld_xb;
#pragma unroll
        for (int nh = 0; nh < G::NH; ++nh) {
          // the 16 x loads of a 128-column block go out together, so their L2 latency is paid once rather than per store
          float2 xo[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) xo[j] = *reinterpret_cast<const float2*>(xr + nh * 128 + 8 * j + cq);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int col = nh * 128 + 8 * j + cq;
            const float y0 = (acc3[nh][4 * j + 2 * h] - mean) * rstd * __ldg(g2 + col) + __ldg(b2 + col);
            const float y1 = (acc3[nh][4 * j + 2 * h + 1] - mean) * rstd * __ldg(g2 + col + 1) + __ldg(b2 + col + 1);
            xo[j].x += y0;
            xo[j].y += y1;
            *reinterpret_cast<float2*>(xr + col) = xo[j];
            *reinterpret_cast<uint32_t*>(xbr + col) = bf16x2(xo[j].x, xo[j].y);
          }
        }
      }
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

// bf16 [rows][cols] row-major with row stride ld (elements): box {64 columns, box_rows}, 128B swizzle, zero OOB fill
int map2d(CUtensorMap* tm, const void* ptr, long long rows, int cols, long long ld, int box_rows) {
  EncodeTiledFn enc = encode_fn();
  if (!enc) return MFR_ERR_CUDA;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || (ld * 2) % 16) return MFR_ERR_ARG;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {64, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[mfr_b200] encoder_tail: cuTensorMapEncodeTiled failed: %d\n", static_cast<int>(r));
    return MFR_ERR_CUDA;
  }
  return MFR_OK;
}

}  // namespace

int encoder_tail_build(const EncoderTailDesc& d, EncoderTailParams* p) {
  if ((d.C != 128 && d.C != 256) || d.n_img < 1 || d.rows_cap < 1) return MFR_ERR_ARG;
  if ((d.ldx & 1) || (d.ld_xb & 1) || (reinterpret_cast<uintptr_t>(d.x) & 7) || (reinterpret_cast<uintptr_t>(d.xb_in) & 15))
    return MFR_ERR_ARG;
  memset(p, 0, sizeof(*p));
  const long long rows = d.rows_cap * d.n_img;
  int rc;
  if ((rc = map2d(&p->tmMsg, d.msg, rows, d.C, d.ld_msg, kRows)) != MFR_OK) return rc;
  if ((rc = map2d(&p->tmX, d.xb_in, rows, d.C, d.ld_xb, kRows)) != MFR_OK) return rc;
  if ((rc = map2d(&p->tmWm, d.w_merge, d.C, d.C, d.C, 128)) != MFR_OK) return rc;
  if ((rc = map2d(&p->tmW0, d.w_mlp0, 2 * d.C, 2 * d.C, 2 * d.C, d.C == 256 ? Cfg<256>::QW : Cfg<128>::QW)) != MFR_OK) return rc;
  if ((rc = map2d(&p->tmW2, d.w_mlp2, d.C, 2 * d.C, 2 * d.C, 128)) != MFR_OK) return rc;
  p->g1 = d.g1; p->b1 = d.b1; p->g2 = d.g2; p->b2 = d.b2;
  p->x = d.x; p->xb = static_cast<unsigned short*>(const_cast<void*>(d.xb_in));
  p->ldx = d.ldx; p->ld_xb = d.ld_xb;
  p->C = d.C; p->n_img = d.n_img; p->rows_cap = d.rows_cap; p->dyn_rows = d.dyn_rows;
  return MFR_OK;
}

int encoder_tail_launch(const EncoderTailParams& p, cudaStream_t st) {
  static bool attr_seen[64] = {};
  if (first_call_on_device(attr_seen)) {
    MFR_CUDA_CHECK(cudaFuncSetAttribute(encoder_tail_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<256>::SMEM));
    MFR_CUDA_CHECK(cudaFuncSetAttribute(encoder_tail_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<128>::SMEM));
  }
  const long long tiles = static_cast<long long>(p.n_img) * ((p.rows_cap + kRows - 1) / kRows);
  // one 225 KB CTA per SM at both widths
  const int grid = static_cast<int>(std::min<long long>(tiles, static_cast<long long>(conv_gemm_num_sms())));
  if (grid <= 0) return MFR_OK;
  if (p.C == 256) encoder_tail_kernel<256><<<grid, kThreads, Cfg<256>::SMEM, st>>>(p);
  else encoder_tail_kernel<128><<<grid, kThreads, Cfg<128>::SMEM, st>>>(p);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

}  // namespace mfr
