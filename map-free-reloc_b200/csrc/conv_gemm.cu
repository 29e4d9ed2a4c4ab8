// wgmma implicit-GEMM convolution kernel (sm_90a). See conv_gemm.cuh for the op definition.
//
// Structure (one persistent CTA per SM, 384 threads = three warpgroups):
//   warp 0          : TMA producer. Per k-block it loads a [TH x TW pixels] x [32 fp32 | 64 bf16 channels] activation
//                     box (rank-4 tensor map over NHWC; halo / padding comes back as zeros through the TMA
//                     out-of-bounds fill, stride-2 through the map's traversal stride) and a [BN filters] x [same
//                     channels] weight box, both 128B-swizzled, into the operand rings.
//   warp 1          : TMA store warp of the compile-time epilogue kinds (epilogue_staged / store_warp).
//   warps 2..3      : idle (they complete the first warpgroup, so that the MMA warpgroups start on a warpgroup
//                     boundary as wgmma requires).
//   warpgroups 1, 2 : MMA + epilogue. Warpgroup g owns rows 64g..64g+63 of every 128-pixel sub-tile: per k-step it
//                     issues one m64nBNk(32 B) wgmma per sub-tile, accumulating in registers; one wgmma group stays in
//                     flight while the slots of the previous one are handed back to the producer. The epilogue
//                     applies alpha / bias / residual / activation to the accumulator registers and either stores
//                     straight to global memory (run-time generic epilogue) or writes a shared-memory staging buffer
//                     that the store warp copies out with TMA stores while the MMA warps go on to the next tile.
// The producer runs ahead by the depth of the rings, so the loads of tile i+1 overlap the epilogue of tile i.
#include "conv_gemm.cuh"
#include "wgmma.cuh"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <mutex>

namespace mfr {

namespace {

constexpr int kMaxSlots = 8;                    // slots per operand ring (A ring and B ring)
constexpr int kBlockK = 32;                     // fp32 elements per k-block = 128 B = swizzle span
constexpr int kTileM = 128;
constexpr int kMaxBN = 256;
constexpr int kAStage = kTileM * kBlockK * 4;   // 16 KB
constexpr int kOperandBytes = 216 * 1024;       // operand rings (A slots + B slots) + the epilogue's staging buffer
constexpr int kZeroBytes = kMaxBN * 32;         // zero page: operand of the unused k-steps of a 32-byte channel-tail group
constexpr int kSmemBytes = kZeroBytes + kOperandBytes + 1024 /*align slack*/;
constexpr int kMmaWarps = 8;                    // two MMA warpgroups
constexpr double kEpiStagedUnit = 250.0;       // cost-model epilogue term of the TMA-store epilogue (choose_cfg)
constexpr int kThreads = 128 + 32 * kMmaWarps;

__device__ __forceinline__ float act_fn(float v, int act, bool fast) {
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  if (act == ACT_LEAKY) return v > 0.f ? v : 0.01f * v;
  if (act == ACT_ELU1) {
    // bf16 outputs: elu(x) + 1 for x <= 0 is exp(x) in (0, 1] — a bare ex2.approx on the pre-scaled argument; its 2-ulp
    // error is far below the bf16 rounding that follows
    if (fast) {
      float e;
      asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fminf(v * 1.4426950408889634f, 0.f)));
      return fmaxf(v, 0.f) + e;
    }
    return v > 0.f ? v + 1.f : __expf(v);
  }
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float bf16_to_float(uint16_t u) { return __uint_as_float(static_cast<uint32_t>(u) << 16); }

// 64-bit wgmma shared-memory matrix descriptor = constant high part | ((address >> 4) & 0x3fff). K-major, 128-byte rows,
// 128B swizzle: 8-row swizzle atoms 1024 B apart (stride byte offset), layout type 1 in bits [62,64).
constexpr uint64_t kDescHi = (1ull << 16) | (64ull << 32) | (1ull << 62);
// same for 32-byte rows with the 32B swizzle (8-row groups 256 B apart, layout type 3): the narrow channel-tail tiles
constexpr uint64_t kDescHi32 = (1ull << 16) | (16ull << 32) | (3ull << 62);

// Epilogue kinds (ConvGemmParams::epi): bit 3 = bf16 output, bit 2 = residual, bits 0-1 = Act; kEpiAny = decided at
// run time per element (act_cols, per-row B operands, odd strides, the other kinds of the tf32 operands)
constexpr int kEpiAny = -1, kEpiOutBf16 = 8, kEpiResidual = 4;
constexpr int epi_kind(bool out_bf16, bool residual, int act) {
  return (out_bf16 ? kEpiOutBf16 : 0) | (residual ? kEpiResidual : 0) | act;
}
// the kinds with their own (TMA-store) instantiations, at BN >= 128: all five with bf16 operands, kF32 with tf32 ones
constexpr int kBf = epi_kind(true, false, ACT_NONE), kBfRelu = epi_kind(true, false, ACT_RELU),
              kBfLeaky = epi_kind(true, false, ACT_LEAKY), kBfResRelu = epi_kind(true, true, ACT_RELU),
              kF32 = epi_kind(false, false, ACT_NONE);
__host__ __device__ constexpr bool staged_inst(int k, int BN, bool bf16) {
  return BN >= 128 && (k == kF32 || (bf16 && (k == kBf || k == kBfRelu || k == kBfLeaky || k == kBfResRelu)));
}

// two neighbouring channels per store: every element offset even and the base pointers aligned accordingly
__host__ __device__ __forceinline__ bool epilogue_vec2(const ConvGemmParams& p) {
  const uintptr_t align = p.out_bf16 ? 3 : 7;
  return ((p.Cout | p.ldo | p.out_y_stride | p.out_img_stride) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.out) & align) == 0 &&
         (p.residual == nullptr ||
          (((p.ldr | p.res_img_stride) & 1) == 0 && (reinterpret_cast<uintptr_t>(p.residual) & align) == 0));
}

// Epilogue of one accumulator fragment: rows (pixels) r0 and r0 + 8 of sub-tile m, columns 8j + 2(lane % 4) + {0, 1}.
template <int BN_T>
__device__ __forceinline__ void epilogue_subtile(const ConvGemmParams& p, const float (&acc)[BN_T / 2], int row0, int lane, int n0,
                                                 int tx, int ty, int img, int m, int tile_rows, int w_lim, bool vec2) {
  const bool obf = p.out_bf16 != 0;
  const float alpha = p.alpha;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + 8 * h;
    const int ly = row / p.TW, lx = row - ly * p.TW;
    const int y = ty * tile_rows + m * p.TH + ly, x = tx * p.TW + lx;
    if (row >= p.TW * p.TH || y >= p.Ho || x >= w_lim) continue;
    const long long o_off = img * p.out_img_stride + static_cast<long long>(y) * p.out_y_stride + static_cast<long long>(x) * p.ldo;
    const long long r_off = img * p.res_img_stride + (static_cast<long long>(y) * p.Wo + x) * p.ldr;
#pragma unroll
    for (int j = 0; j < BN_T / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      const int n = n0 + c;
      if (c >= p.BN || n >= p.Cout) continue;
      float v[2] = {acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]};
      const bool two = n + 1 < p.Cout;
      if (vec2 && two) {
        float b0 = 0.f, b1 = 0.f;
        if (p.bias != nullptr) { b0 = __ldg(p.bias + n); b1 = __ldg(p.bias + n + 1); }
        v[0] = fmaf(v[0], alpha, b0);
        v[1] = fmaf(v[1], alpha, b1);
        if (p.residual != nullptr) {
          if (obf) {
            const uint32_t r = __ldg(reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(p.residual) + r_off + n));
            v[0] += __uint_as_float(r << 16);
            v[1] += __uint_as_float(r & 0xffff0000u);
          } else {
            const float2 r = __ldg(reinterpret_cast<const float2*>(p.residual + r_off + n));
            v[0] += r.x;
            v[1] += r.y;
          }
        }
        if (n < p.act_cols) v[0] = act_fn(v[0], p.act, obf);
        if (n + 1 < p.act_cols) v[1] = act_fn(v[1], p.act, obf);
        if (obf) *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + o_off + n) = pack_bf16x2(v[0], v[1]);
        else *reinterpret_cast<float2*>(p.out + o_off + n) = make_float2(v[0], v[1]);
      } else {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int ne = n + e;
          if (ne >= p.Cout || c + e >= p.BN) continue;
          float t = v[e] * alpha;
          if (p.bias != nullptr) t += __ldg(p.bias + ne);
          if (p.residual != nullptr)
            t += obf ? bf16_to_float(reinterpret_cast<const uint16_t*>(p.residual)[r_off + ne]) : __ldg(p.residual + r_off + ne);
          if (ne < p.act_cols) t = act_fn(t, p.act, obf);
          if (obf) reinterpret_cast<uint16_t*>(p.out)[o_off + ne] = static_cast<uint16_t>(pack_bf16x2(t, 0.f) & 0xffffu);
          else p.out[o_off + ne] = t;
        }
      }
    }
  }
}

// Staging layout of the TMA-store epilogue. A CTA tile leaves shared memory as boxes {kCW channels, TW, TH, 1}: box
// b = m * nbox + c holds channel chunk c of sub-tile m, 128 rows (pixel ly * TW + lx) of 128 bytes, 128B-swizzled; a
// BN that is not a multiple of kCW (200) ends in a narrow box of BN % kCW channels, unswizzled rows (tmO2 / tmR2). The
// boxes are placed in order into passes of at most kStageMax bytes: one pass for every bf16 tile, two for the larger fp32
// tiles. stage_place packs (pass << 16) | byte offset in the staging buffer.
constexpr int kStageMax = 64 * 1024;
constexpr int kBox = kTileM * 128;   // one full box
__host__ __device__ constexpr int stage_cw(bool bf16) { return bf16 ? 64 : 32; }
__host__ __device__ constexpr int stage_nbox(int BN, bool bf16) { return (BN + stage_cw(bf16) - 1) / stage_cw(bf16); }
__host__ __device__ constexpr int stage_narrow_row(int BN, bool bf16) { return (BN % stage_cw(bf16)) * (bf16 ? 2 : 4); }
__host__ __device__ constexpr int stage_box_bytes(int BN, bool bf16, int c) {
  return (c + 1) * stage_cw(bf16) <= BN ? kBox : kTileM * stage_narrow_row(BN, bf16);
}
__host__ __device__ constexpr int stage_place(int BN, bool bf16, int b) {
  int pass = 0, off = 0;
  for (int i = 0;; ++i) {
    const int sz = stage_box_bytes(BN, bf16, i % stage_nbox(BN, bf16));
    if (off + sz > kStageMax) { ++pass; off = 0; }
    if (i == b) return (pass << 16) | off;
    off += sz;
  }
}
// staging bytes of a tile (its first and largest pass)
__host__ __device__ constexpr int stage_bytes(int BN, bool bf16, int MT) {
  int bytes = 0;
  for (int b = 0; b < MT * stage_nbox(BN, bf16); ++b)
    if ((stage_place(BN, bf16, b) >> 16) == 0) bytes = (stage_place(BN, bf16, b) & 0xffff) + stage_box_bytes(BN, bf16, b % stage_nbox(BN, bf16));
  return bytes;
}

// Epilogue with the output type, residual and activation fixed at compile time (EPI = epi_kind(...)): the kinds of the
// ResNet-FPN convs, the coarse q|k|v projections and the correlation. The MMA warps apply alpha / bias / residual /
// activation to the accumulators and write the result into the staging buffer (bf16 through stmatrix, fp32 as 8-byte
// vectors); the store warp copies it out with TMA stores, whose tensor map clips ragged tiles and the channels >= Cout.
// A residual has been loaded into the staging buffer by the store warp (zero outside the tensor) and is read from the
// positions the result then overwrites. Per pass: wait for the buffer (st_empty), fill it, fence + barrier over the 256
// MMA threads, hand it to the store warp (st_full).
template <int BN_T, int MT_T, int EPI>
__device__ __forceinline__ void epilogue_staged(const ConvGemmParams& p, const float (&acc)[MT_T][BN_T / 2], uint32_t stage,
                                                uint32_t st_empty, uint32_t st_full, int tile_index, int row_base,
                                                int lane, int n0) {
  constexpr bool kOutBf16 = (EPI & kEpiOutBf16) != 0, kRes = (EPI & kEpiResidual) != 0;
  constexpr int kAct = EPI & 3;
  constexpr int kNBox = stage_nbox(BN_T, kOutBf16), kCW = stage_cw(kOutBf16);
  constexpr int kPasses = (stage_place(BN_T, kOutBf16, MT_T * kNBox - 1) >> 16) + 1;
  static_assert(!kRes || (kOutBf16 && kPasses == 1), "a residual is staged in one pass");
  const float alpha = p.alpha;
  const int q = lane & 3;
  auto bias2 = [&](int n) {   // columns n, n + 1 (Cout is even); the columns of a tile beyond Cout are clipped by the store
    return (p.bias != nullptr && n < p.Cout) ? __ldg(reinterpret_cast<const float2*>(p.bias + n)) : make_float2(0.f, 0.f);
  };
#pragma unroll
  for (int pass = 0; pass < kPasses; ++pass) {
    mbar_wait_inl(st_empty, static_cast<uint32_t>(tile_index * kPasses + pass) & 1u, 7);
    if constexpr (kOutBf16) {
      // stmatrix / ldmatrix x4 over columns 8j .. 8j + 15: matrix i = (column group j + i / 2, row half i % 2), whose
      // row addresses come from lanes 8i .. 8i + 7; x2 for a last odd column group
      const int mi = lane >> 3;
      const int arow = row_base + (lane & 7) + 8 * (mi & 1);
#pragma unroll
      for (int j = 0; j < BN_T / 8; j += 2) {
        const bool two = j + 1 < BN_T / 8;
        float2 bb[2];
#pragma unroll
        for (int t = 0; t < 2; ++t) bb[t] = (j + t < BN_T / 8) ? bias2(n0 + 8 * (j + t) + 2 * q) : make_float2(0.f, 0.f);
#pragma unroll
        for (int m = 0; m < MT_T; ++m) {
          const int c = (8 * j) / kCW, b = m * kNBox + c;
          const uint32_t box = stage + (stage_place(BN_T, true, b) & 0xffff);
          const int acol = 8 * j + (two ? 8 * (mi >> 1) : 0) - c * kCW;
          const uint32_t addr = (c + 1) * kCW <= BN_T ? sw_addr(box, arow, acol, 0)
                                                      : box + static_cast<uint32_t>(arow * stage_narrow_row(BN_T, true));
          uint32_t r[4] = {0u, 0u, 0u, 0u};
          if constexpr (kRes) {
            if (two) ldsm_x4(addr, r[0], r[1], r[2], r[3]);
            else ldsm_x2(addr, r[0], r[1]);
          }
          uint32_t o[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int jj = j + (i >> 1), h = i & 1;
            if (jj >= BN_T / 8) { o[i] = 0u; continue; }
            float v0 = fmaf(acc[m][4 * jj + 2 * h], alpha, bb[i >> 1].x), v1 = fmaf(acc[m][4 * jj + 2 * h + 1], alpha, bb[i >> 1].y);
            if constexpr (kRes) {
              v0 += __uint_as_float(r[i] << 16);
              v1 += __uint_as_float(r[i] & 0xffff0000u);
            }
            o[i] = pack_bf16x2(act_fn(v0, kAct, true), act_fn(v1, kAct, true));
          }
          if (two) stsm_x4(addr, o[0], o[1], o[2], o[3]);
          else stsm_x2(addr, o[0], o[1]);
        }
      }
    } else {
      const int row0 = row_base + (lane >> 2);
#pragma unroll
      for (int j = 0; j < BN_T / 8; ++j) {
        const float2 bb = bias2(n0 + 8 * j + 2 * q);
#pragma unroll
        for (int m = 0; m < MT_T; ++m) {
          const int c = (8 * j) / kCW, b = m * kNBox + c;
          if ((stage_place(BN_T, false, b) >> 16) != pass) continue;
          const uint32_t box = stage + (stage_place(BN_T, false, b) & 0xffff);
          const int col = 8 * j + 2 * q - c * kCW;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = row0 + 8 * h;
            const uint32_t addr = (c + 1) * kCW <= BN_T ? sw_addr(box, row, 2 * col, 0)
                                                        : box + static_cast<uint32_t>(row * stage_narrow_row(BN_T, false) + 4 * col);
            const float v0 = act_fn(fmaf(acc[m][4 * j + 2 * h], alpha, bb.x), kAct, false);
            const float v1 = act_fn(fmaf(acc[m][4 * j + 2 * h + 1], alpha, bb.y), kAct, false);
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v0), "f"(v1) : "memory");
          }
        }
      }
    }
    fence_proxy_async_smem();   // the staging buffer is read by the TMA store (async proxy)
    named_bar_sync(1, 32 * kMmaWarps);
    if (threadIdx.x == 128) mbar_arrive(st_full);
  }
}

// Store warp of the TMA-store epilogue: per pass of every tile it waits for the staging buffer, stores its boxes, and
// once the stores have read it hands it back -- for the residual kind after loading the next tile's residual into it.
// With a device row count (w_lim < Wo; H = 1, no residual) the output map still ends at Wo, so the one tile per image
// that crosses w_lim is copied out by the warp itself, its live rows only: no row at or past w_lim is written.
template <int BN_T, int MT_T, int EPI>
__device__ __forceinline__ void store_warp(const ConvGemmParams& p, uint32_t stage, uint32_t st_empty, uint32_t st_full,
                                           int total_tiles, int tiles_x, int tile_rows, int w_lim) {
  constexpr bool kOutBf16 = (EPI & kEpiOutBf16) != 0, kRes = (EPI & kEpiResidual) != 0;
  constexpr int kNBox = stage_nbox(BN_T, kOutBf16), kCW = stage_cw(kOutBf16);
  constexpr int kPasses = (stage_place(BN_T, kOutBf16, MT_T * kNBox - 1) >> 16) + 1;
  constexpr int kOsz = kOutBf16 ? 2 : 4;
  // a device row count comes with H = 1, so MT = 1, and without a residual: only those instantiations handle it
  constexpr bool kDynRows = MT_T == 1 && !kRes;
  const int x_lim = kDynRows ? w_lim : p.Wo;
  struct Tile { int n0, x0, y0, img; };
  auto tile_of = [&](int item) {
    int mt, nt;
    if (p.nt_fast) { mt = item / p.n_tiles; nt = item - mt * p.n_tiles; }
    else { nt = item / (p.N * p.tiles_y * tiles_x); mt = item - nt * (p.N * p.tiles_y * tiles_x); }
    const int tx = mt % tiles_x, ty = (mt / tiles_x) % p.tiles_y;
    return Tile{nt * p.BN, tx * p.TW, ty * tile_rows, mt / (tiles_x * p.tiles_y)};
  };
  // the staging buffer is free for the next pass; with a residual: load the residual boxes of tile t into it
  auto hand_back = [&](const Tile& t) {
    if constexpr (kRes) {
      if (elect_one_sync()) {
        uint32_t bytes = 0;
#pragma unroll
        for (int b = 0; b < MT_T * kNBox; ++b)
          if (t.y0 + (b / kNBox) * p.TH < p.Ho) bytes += static_cast<uint32_t>(p.TW * p.TH * ((b % kNBox + 1) * kCW <= BN_T ? 128 : stage_narrow_row(BN_T, true)));
        mbar_arrive_expect_tx(st_empty, bytes);
#pragma unroll
        for (int b = 0; b < MT_T * kNBox; ++b) {
          const int m = b / kNBox, c = b % kNBox;
          if (t.y0 + m * p.TH >= p.Ho) continue;
          tma_load_4d(stage + (stage_place(BN_T, true, b) & 0xffff), (c + 1) * kCW <= BN_T ? &p.tmR : &p.tmR2, st_empty,
                      t.n0 + c * kCW, t.x0, t.y0 + m * p.TH, t.img);
        }
      }
    } else {
      if (elect_one_sync()) mbar_arrive(st_empty);
    }
    __syncwarp();
  };
  if (static_cast<int>(blockIdx.x) < total_tiles) hand_back(tile_of(blockIdx.x));
  uint32_t parity = 0;
  for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
    const Tile t = tile_of(item);
    const bool part = kDynRows && x_lim < p.Wo && t.x0 + p.TW > x_lim;   // crosses the device row count
#pragma unroll
    for (int pass = 0; pass < kPasses; ++pass) {
      mbar_wait_inl(st_full, parity, 8);
      parity ^= 1u;
      if (!part) {
        if (elect_one_sync()) {
#pragma unroll
          for (int b = 0; b < MT_T * kNBox; ++b) {
            const int m = b / kNBox, c = b % kNBox;
            if ((stage_place(BN_T, kOutBf16, b) >> 16) != pass || t.y0 + m * p.TH >= p.Ho) continue;
            tma_store_4d((c + 1) * kCW <= BN_T ? &p.tmO : &p.tmO2, stage + (stage_place(BN_T, kOutBf16, b) & 0xffff),
                         t.n0 + c * kCW, t.x0, t.y0 + m * p.TH, t.img);
          }
          tma_store_commit();
        }
      } else if constexpr (kDynRows) {
        // the live rows' channels below p.cout_tma, one 16-byte group per lane, un-swizzled from the staging buffer
        static_assert(stage_narrow_row(BN_T, kOutBf16) % 16 == 0, "the narrow box holds whole 16-byte groups");
        const int c_hi = min(p.cout_tma - t.n0, BN_T);
#pragma unroll
        for (int b = 0; b < MT_T * kNBox; ++b) {
          const int m = b / kNBox, c = b % kNBox;
          if ((stage_place(BN_T, kOutBf16, b) >> 16) != pass || t.y0 + m * p.TH >= p.Ho) continue;
          const uint32_t box = stage + (stage_place(BN_T, kOutBf16, b) & 0xffff);
          const bool full = (c + 1) * kCW <= BN_T;
          const int groups = full ? 8 : stage_narrow_row(BN_T, kOutBf16) / 16;   // 16-byte groups per box row
          for (int i = static_cast<int>(threadIdx.x & 31); i < p.TW * p.TH * groups; i += 32) {
            const int row = i / groups, g = i - row * groups, cl = c * kCW + g * (16 / kOsz);
            const int ly = row / p.TW, y = t.y0 + m * p.TH + ly, x = t.x0 + row - ly * p.TW;
            if (cl >= c_hi || y >= p.Ho || x >= x_lim) continue;
            const uint32_t addr = full ? box + static_cast<uint32_t>(row * 128 + ((g ^ (row & 7)) << 4))
                                       : box + static_cast<uint32_t>(row * stage_narrow_row(BN_T, kOutBf16) + 16 * g);
            uint4 v;
            asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
            const long long o = t.img * p.out_img_stride + static_cast<long long>(y) * p.out_y_stride + static_cast<long long>(x) * p.ldo + t.n0 + cl;
            *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(p.out) + o * kOsz) = v;
          }
        }
      }
      // TMA stores write whole 16-byte groups of channels: the output map ends at p.cout_tma (Cout rounded down to 16
      // bytes), and the warp copies the channels from there to Cout (196 = 192 + 4) with plain stores
      if (p.cout_tma < p.Cout) {
        const int c_lo = max(p.cout_tma - t.n0, 0), c_hi = min(p.Cout - t.n0, BN_T);
        for (int m = 0; m < MT_T; ++m)
          for (int row = static_cast<int>(threadIdx.x & 31); row < p.TW * p.TH; row += 32) {
            const int ly = row / p.TW, y = t.y0 + m * p.TH + ly, x = t.x0 + row - ly * p.TW;
            if (y >= p.Ho || x >= x_lim) continue;
            const long long o = t.img * p.out_img_stride + static_cast<long long>(y) * p.out_y_stride + static_cast<long long>(x) * p.ldo + t.n0;
            for (int cl = c_lo; cl < c_hi; cl += 2) {
              const int c = cl / kCW, b = m * kNBox + c;
              if ((stage_place(BN_T, kOutBf16, b) >> 16) != pass) continue;
              const uint32_t box = stage + (stage_place(BN_T, kOutBf16, b) & 0xffff);
              const int cc = cl - c * kCW;
              const uint32_t addr = (c + 1) * kCW <= BN_T ? sw_addr(box, row, kOutBf16 ? cc : 2 * cc, 0)
                                                          : box + static_cast<uint32_t>(row * stage_narrow_row(BN_T, kOutBf16) + cc * (kOutBf16 ? 2 : 4));
              if constexpr (kOutBf16) {
                uint32_t v;
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
                *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.out) + o + cl) = v;
              } else {
                float2 v;
                asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr) : "memory");
                *reinterpret_cast<float2*>(p.out + o + cl) = v;
              }
            }
          }
      }
      if (elect_one_sync()) tma_store_wait_read();
      __syncwarp();
      if (pass + 1 < kPasses) hand_back(t);
      else if (item + static_cast<int>(gridDim.x) < total_tiles) hand_back(tile_of(item + gridDim.x));
    }
  }
  if (elect_one_sync()) tma_store_wait_all();
  __syncwarp();
}

// BN_T = N tile (wgmma N), MT_T = 128-pixel sub-tiles per CTA tile, BF16 = operand type, EPI = epilogue kind (kEpiAny:
// the run-time generic epilogue); the host launches the instantiation equal to (p.BN, p.MT, p.in_bf16, p.epi), and
// conv_gemm_build only names a kind in p.epi that has one (staged_inst). Between the wgmma instructions of a group
// there is no control flow (ptxas would otherwise serialise them): every k-block issues 4 k-steps, the channel tail of
// a 128-byte k-block is zero-filled by TMA, and the 3 unused k-steps of a 32-byte tail group read the zero page.
template <int BN_T, int MT_T, bool BF16, int EPI>
__global__ void __launch_bounds__(kThreads, 1) conv_gemm_kernel(const __grid_constant__ ConvGemmParams p) {
  static_assert(EPI == kEpiAny || staged_inst(EPI, BN_T, BF16), "no TMA-store epilogue for this kind");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t s_bars[4 * kMaxSlots + 2];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t smem_zero = smem_base;
  const uint32_t smem_a = smem_base + kZeroBytes;
  const uint32_t smem_b = smem_a + p.a_slots * p.a_slot_bytes;
  const uint32_t stage = smem_a + kOperandBytes - p.stage_bytes;   // TMA-store epilogue: the top of the operand space
  const uint32_t bar_base = smem_u32(s_bars);
  // barriers: a_full[8], a_empty[8], b_full[8], b_empty[8]. Generic mode uses one ring (A and B tile of a k-block share
  // slot and barriers: the "a" set); halo mode uses both rings. An empty barrier completes when every MMA warp released it.
  auto a_full = [&](int s) { return bar_base + 8u * s; };
  auto a_empty = [&](int s) { return bar_base + 8u * (kMaxSlots + s); };
  auto b_full = [&](int s) { return bar_base + 8u * (2 * kMaxSlots + s); };
  auto b_empty = [&](int s) { return bar_base + 8u * (3 * kMaxSlots + s); };
  const uint32_t st_empty = bar_base + 8u * (4 * kMaxSlots), st_full = st_empty + 8u;   // staging buffer free / filled

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);   // warp-uniform role
  const int lane = threadIdx.x & 31;

  for (int i = threadIdx.x; i < kZeroBytes / 16; i += blockDim.x)
    asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(smem_zero + 16u * i), "r"(0u) : "memory");
  fence_proxy_async_smem();   // the zero page is read by wgmma (async proxy)
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmA);
    tma_prefetch_desc(&p.tmB);
    if constexpr (EPI != kEpiAny) {
      mbar_init(st_empty, 1);
      mbar_init(st_full, 1);
    }
    for (int s = 0; s < kMaxSlots; ++s) {
      mbar_init(a_full(s), 1);
      mbar_init(a_empty(s), kMmaWarps);
      mbar_init(b_full(s), 1);
      mbar_init(b_empty(s), kMmaWarps);
    }
    fence_barrier_init();
  }
  __syncthreads();

  int w_lim = p.Wo, tiles_x = p.tiles_x;
  if (p.dyn_w != nullptr) {
    w_lim = min(p.Wo, *p.dyn_w);
    tiles_x = (w_lim + p.TW - 1) / p.TW;
  }
  const int m_tiles = p.N * p.tiles_y * tiles_x;
  const int total_tiles = m_tiles * p.n_tiles;
  const int tile_rows = MT_T * p.TH;          // output rows of one CTA tile
  auto item_tile = [&](int item, int& mt, int& nt) {
    if (p.nt_fast) {   // the N tiles of a pixel tile run at the same time on neighbouring SMs: its A tiles are read from DRAM once
      mt = item / p.n_tiles;
      nt = item - mt * p.n_tiles;
    } else {
      nt = item / m_tiles;
      mt = item - nt * m_tiles;
    }
  };
  const int kb_per_tap = p.kb_per_tap, kblk = p.kblk, R = p.R, S = p.S;
  const int a_slots = p.a_slots, b_slots = p.b_slots;
  const uint32_t a_slot_bytes = p.a_slot_bytes, a_bytes = p.a_bytes, b_bytes = p.b_bytes;

  if (warp == 0) {
    // ------------------------------------------------------------------ TMA producer
    int sa = 0, sb = 0;
    uint32_t pa = 0, pb = 0;
    for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
      int mt, nt;
      item_tile(item, mt, nt);
      const int tx = mt % tiles_x;
      const int ty = (mt / tiles_x) % p.tiles_y;
      const int img = mt / (tiles_x * p.tiles_y);
      const int x_in0 = tx * p.TW * p.stride - p.pad;
      const int y_in0 = ty * tile_rows * p.stride - p.pad;
      const int n0 = nt * p.BN;
      if (p.halo) {
        for (int cb = 0; cb < kb_per_tap; ++cb) {
          const int c0 = cb * kblk;
          const bool tail = p.tail32 && cb == kb_per_tap - 1;       // narrow boxes for the channel tail
          const CUtensorMap* tmA = tail ? &p.tmA2 : &p.tmA;
          const CUtensorMap* tmB = tail ? &p.tmB2 : &p.tmB;
          const uint32_t ab = tail ? p.a_bytes2 : a_bytes, bb = tail ? p.b_bytes2 : b_bytes;
          // B tiles in the order the taps are summed; the A box of column kx goes ahead of its first tap (ky = 0)
          for (int g = 0; g < 9; ++g) {
            const int kx = p.kx_major ? g / 3 : g % 3, ky = p.kx_major ? g % 3 : g / 3;
            if (ky == 0) {
              mbar_wait_inl(a_empty(sa), pa ^ 1u, 1);
              if (elect_one_sync()) {
                mbar_arrive_expect_tx(a_full(sa), ab);
                tma_load_4d(smem_a + sa * a_slot_bytes, tmA, a_full(sa), c0, x_in0 + kx, y_in0, img);
              }
              if (++sa == a_slots) { sa = 0; pa ^= 1u; }
            }
            mbar_wait_inl(b_empty(sb), pb ^ 1u, 5);
            if (elect_one_sync()) {
              mbar_arrive_expect_tx(b_full(sb), bb);
              tma_load_3d(smem_b + sb * b_bytes, tmB, b_full(sb), c0, ky * 3 + kx, n0);
            }
            if (++sb == b_slots) { sb = 0; pb ^= 1u; }
          }
        }
      } else {
        const int bz = p.b_batched ? img : -1;
        for (int cb = 0; cb < kb_per_tap; ++cb) {
          const int c0 = cb * kblk;
          const bool tail = p.tail32 && cb == kb_per_tap - 1;
          const CUtensorMap* tmA = tail ? &p.tmA2 : &p.tmA;
          const CUtensorMap* tmB = tail ? &p.tmB2 : &p.tmB;
          const uint32_t ab = tail ? p.a_bytes2 + p.b_bytes2 : a_bytes + b_bytes;
          // taps in the order they are summed (p.kx_major)
          for (int t = 0; t < R * S; ++t) {
            const int ky = p.kx_major ? t % R : t / S, kx = p.kx_major ? t / R : t % S, tap = ky * S + kx;
            mbar_wait_inl(a_empty(sa), pa ^ 1u, 1);
            if (elect_one_sync()) {
              mbar_arrive_expect_tx(a_full(sa), ab);
              if (p.a_yx) tma_load_4d(smem_a + sa * a_slot_bytes, tmA, a_full(sa), c0, y_in0 + ky, x_in0 + kx, img);
              else tma_load_4d(smem_a + sa * a_slot_bytes, tmA, a_full(sa), c0, x_in0 + kx, y_in0 + ky, img);
              if (p.b_batched == 2) {
                if (p.b_yx) tma_load_4d(smem_b + sa * b_bytes, tmB, a_full(sa), c0, ty, n0, img ^ p.b_xor);
                else tma_load_4d(smem_b + sa * b_bytes, tmB, a_full(sa), c0, n0, ty, img ^ p.b_xor);
              }
              else tma_load_3d(smem_b + sa * b_bytes, tmB, a_full(sa), c0, bz >= 0 ? bz : tap, n0);
            }
            if (++sa == a_slots) { sa = 0; pa ^= 1u; }
          }
        }
      }
    }
  } else if (warp == 1) {
    // ------------------------------------------------------------------ TMA store warp
    if constexpr (EPI != kEpiAny) store_warp<BN_T, MT_T, EPI>(p, stage, st_empty, st_full, total_tiles, tiles_x, tile_rows, w_lim);
  } else if (warp >= 4) {
    // ------------------------------------------------------------------ MMA + epilogue warpgroups
    const int wg = (warp - 4) >> 2;                   // rows 64 wg .. 64 wg + 63 of each sub-tile
    const int row0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    const uint32_t sub_bytes = static_cast<uint32_t>(p.TH * p.TW * 128);   // A bytes of one 128-row sub-tile
    const uint32_t ky_bytes = static_cast<uint32_t>(p.TW * 128);           // one halo row
    const bool vec2 = epilogue_vec2(p);
    float acc[MT_T][BN_T / 2];
    int sa = 0, sb = 0;
    uint32_t pa = 0, pb = 0;
    // slots of the wgmma group still in flight (-1: none): released once the next group is issued and this one has
    // completed
    int rel_a = -1, rel_b = -1;
    auto release = [&]() {
      if (rel_a < 0 && rel_b < 0) return;
      __syncwarp();
      if (lane == 0) {
        if (rel_a >= 0) mbar_arrive(a_empty(rel_a));
        if (rel_b >= 0) mbar_arrive(b_empty(rel_b));
      }
      rel_a = rel_b = -1;
    };
    auto mma = [&](float (&d)[BN_T / 2], uint64_t adesc, uint64_t bdesc) {
      if constexpr (BF16) wgmma_bf16<BN_T>(d, adesc, bdesc);
      else wgmma_tf32<BN_T>(d, adesc, bdesc);
    };
    const uint64_t zdesc = kDescHi32 | ((smem_zero >> 4) & 0x3fffu);
    // k-step k of a group whose step 0 is (adesc, bdesc): +32 B of K = +2 in the address field; a tail group has one step
    auto kdesc = [&](uint64_t d, int k, bool tail) { return (tail && k > 0) ? zdesc : d + 2 * k; };
    for (int item = blockIdx.x; item < total_tiles; item += gridDim.x) {
      int mt, nt;
      item_tile(item, mt, nt);
#pragma unroll
      for (int m = 0; m < MT_T; ++m)
#pragma unroll
        for (int i = 0; i < BN_T / 2; ++i) acc[m][i] = 0.f;
      if (p.halo) {
        for (int cb = 0; cb < kb_per_tap; ++cb) {
          const bool tail = p.tail32 && cb == kb_per_tap - 1;   // 32-byte rows: one k-step, 32B-swizzle descriptors
          const uint64_t dhi = tail ? kDescHi32 : kDescHi;
          const uint32_t row_b = tail ? 32u : 128u;
          const uint32_t subb = tail ? sub_bytes >> 2 : sub_bytes, kyb = tail ? ky_bytes >> 2 : ky_bytes;
          // one wgmma group per tap, in the tap order of p.kx_major: its B slot goes back as soon as the group has
          // completed (4 B slots keep the producer ahead at BN = 256); the A slot of column kx (slot sa + kx of the
          // ring) goes back with its third tap
#pragma unroll 1
          for (int g = 0; g < 9; ++g) {
            const int kx = p.kx_major ? g / 3 : g % 3, ky = p.kx_major ? g % 3 : g / 3;
            int sx = sa + kx;
            uint32_t px = pa;
            if (sx >= a_slots) { sx -= a_slots; px ^= 1u; }
            if (ky == 0) mbar_wait_inl(a_full(sx), px, 3);
            mbar_wait_inl(b_full(sb), pb, 6);
            const uint32_t a_slot = smem_a + sx * a_slot_bytes + static_cast<uint32_t>(64 * wg) * row_b;
            const uint64_t bdesc = dhi | (((smem_b + sb * b_bytes) >> 4) & 0x3fffu);
            wgmma_fence();
#pragma unroll
            for (int m = 0; m < MT_T; ++m) {
              const uint64_t adesc = dhi | (((a_slot + m * subb + ky * kyb) >> 4) & 0x3fffu);
#pragma unroll
              for (int k = 0; k < 4; ++k) mma(acc[m], kdesc(adesc, k, tail), kdesc(bdesc, k, tail));
            }
            wgmma_commit();
            wgmma_wait<1>();
            release();
            rel_a = ky == 2 ? sx : -1; rel_b = sb;
            if (++sb == b_slots) { sb = 0; pb ^= 1u; }
          }
          sa += 3;
          while (sa >= a_slots) { sa -= a_slots; pa ^= 1u; }
        }
      } else {
        const int num_kb = R * S * kb_per_tap, taps = R * S;
        int tap = 0, cb = 0;
        for (int i = 0; i < num_kb; ++i) {
          mbar_wait_inl(a_full(sa), pa, 3);
          const bool tail = p.tail32 && cb == kb_per_tap - 1;
          const uint64_t dhi = tail ? kDescHi32 : kDescHi;
          const uint64_t bdesc = dhi | (((smem_b + sa * b_bytes) >> 4) & 0x3fffu);
          const uint32_t a_slot = smem_a + sa * a_slot_bytes + static_cast<uint32_t>(64 * wg) * (tail ? 32u : 128u);
          wgmma_fence();
#pragma unroll
          for (int m = 0; m < MT_T; ++m) {
            const uint64_t adesc = dhi | (((a_slot + m * (tail ? sub_bytes >> 2 : sub_bytes)) >> 4) & 0x3fffu);
#pragma unroll
            for (int k = 0; k < 4; ++k) mma(acc[m], kdesc(adesc, k, tail), kdesc(bdesc, k, tail));
          }
          wgmma_commit();
          wgmma_wait<1>();
          release();
          rel_a = sa;
          if (++sa == a_slots) { sa = 0; pa ^= 1u; }
          if (++tap == taps) { tap = 0; ++cb; }
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int m = 0; m < MT_T; ++m) wgmma_fence_regs(acc[m]);
      release();
      if constexpr (EPI == kEpiAny) {
        const int tx = mt % tiles_x;
        const int ty = (mt / tiles_x) % p.tiles_y;
        const int img = mt / (tiles_x * p.tiles_y);
#pragma unroll
        for (int m = 0; m < MT_T; ++m)
          epilogue_subtile<BN_T>(p, acc[m], row0, lane, nt * p.BN, tx, ty, img, m, tile_rows, w_lim, vec2);
      } else {
        // staging address and barriers recomputed here: nothing extra stays live across the main loop
        const uint32_t stage_ = ((smem_u32(smem_raw) + 1023u) & ~1023u) + kZeroBytes + kOperandBytes - p.stage_bytes;
        const uint32_t bars = smem_u32(s_bars) + 8u * (4 * kMaxSlots);
        epilogue_staged<BN_T, MT_T, EPI>(p, acc, stage_, bars, bars + 8u, (item - static_cast<int>(blockIdx.x)) / static_cast<int>(gridDim.x),
                                         row0 - (lane >> 2), lane, nt * p.BN);
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) ==
            cudaSuccess &&
        qres == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(f);
    }
  });
  return fn;
}

// Tiling of one op: output tile = MT sub-tiles of TW x TH (<= 128) pixels, BN output channels.
struct TileCfg {
  int TW, TH, MT, BN, n_tiles, halo;
  double cost;
};

// N tiles the kernel is instantiated for (the wgmma N of one instruction)
int bn_for(int cols) {
  for (int bn : {32, 64, 128, 200}) if (cols <= bn) return bn;
  return 256;
}

// Relative cost model used to pick the tiling (units ~ ns per CTA tile). The constants are estimates, not measured on
// an H100; only the ranking of the candidate tilings matters:
//   MMA      : one 128 x BN x (32 B of K) step, issued as two m64 wgmma, ~ 30 + 0.25 * BN; every wgmma group waits for
//              its predecessor, ~ 200 per group; a k-block always issues 4 steps
//   feed     : operand bytes through L2 -> shared memory at ~ 100 bytes per unit per SM when all SMs pull at once
//   epilogue : ~ 500 per 32-channel chunk of a 128-pixel sub-tile (run-time generic epilogue), kEpiStagedUnit with the
//              TMA-store epilogue
// times the number of waves of tiles over the SMs.
struct RingCfg { int a_slots, b_slots, a_slot_bytes; };
// ring_bytes: what the staging buffer of the TMA-store epilogue leaves of kOperandBytes
RingCfg ring_cfg(int halo, bool kx_major, int MT, int TW, int TH, int BN, int ring_bytes) {
  RingCfg r{};
  const int b_bytes = BN * 128;
  if (halo) {
    // 3 A slots and >= 6 B slots (two kx groups of B tiles in flight) where they fit, else 2 A slots, else the
    // least that keeps one group in flight while the next one loads: 4 B slots (BN > 128). Summed ky-major, a k-block
    // holds the A boxes of all three columns at once: 3 A slots at least.
    r.a_slot_bytes = TW * (MT * TH + 2) * 128;   // multiple of 1 KB (TW % 8 == 0)
    for (int min_b : {6, 4}) {
      for (int a = 3; a >= (kx_major ? 2 : 3); --a) {
        r.a_slots = a;
        r.b_slots = std::min(kMaxSlots, (ring_bytes - a * r.a_slot_bytes) / b_bytes);
        if (r.b_slots >= min_b) return r;
      }
    }
  } else {
    // generic mode pads the A slot to whole 128-row sub-tiles (the MMA reads 128 rows regardless)
    r.a_slot_bytes = std::max((TW * TH * MT * 128 + 1023) / 1024 * 1024, MT * kAStage);
    r.a_slots = r.b_slots = std::min(kMaxSlots, ring_bytes / (r.a_slot_bytes + b_bytes));
  }
  return r;
}

// staging bytes of the TMA-store epilogue (staged: -1 none, 0 fp32, 1 bf16 output; only the BN >= 128 tiles have it)
int staging_for(int staged, int MT, int BN) { return (staged >= 0 && BN >= 128) ? stage_bytes(BN, staged != 0, MT) : 0; }

TileCfg choose_cfg(int N, int Ho, int Wo, int Cout, int R, int S, int stride, int pad, int kb_per_tap,
                   bool tail32, bool kx_major, bool allow_mt2, bool single_row_tiles, int staged) {
  const int sms = conv_gemm_num_sms();
  const int c8 = (Cout + 7) / 8 * 8;
  const int taps = R * S;
  const int ksteps_tap = kb_per_tap * 4;
  const bool can_halo = R == 3 && S == 3 && stride == 1 && pad == 1;
  TileCfg best{};
  best.cost = 1e300;
  // test hook: MFR_CONV_FORCE="halo,MT,TW" restricts the search (-1 = free); unusable values fall back to free
  int f_halo = -1, f_mt = -1, f_tw = -1;
  if (const char* e = getenv("MFR_CONV_FORCE")) sscanf(e, "%d,%d,%d", &f_halo, &f_mt, &f_tw);
  for (int pass = 0; pass < 2 && best.cost > 1e299; ++pass) {
  if (pass == 1) f_halo = f_mt = f_tw = -1;
  const int nt0 = (c8 + kMaxBN - 1) / kMaxBN;
  for (int nt = nt0; nt <= nt0 * 4; nt *= 2) {
    const int BN = bn_for((c8 + nt - 1) / nt);
    if (nt > nt0 && BN < 64) break;
    for (int halo = 0; halo <= (can_halo ? 1 : 0); ++halo) {
      for (int MT = 1; MT <= 2; ++MT) {
        if (MT == 2 && (BN > 128 || Ho == 1 || !allow_mt2)) continue;
        if ((f_halo >= 0 && halo != f_halo) || (f_mt > 0 && MT != f_mt)) continue;
        for (int tw = 1; tw <= 128; ++tw) {
          if (f_tw > 0 && tw != f_tw) continue;
          if (halo && (tw % 8 != 0 || 128 % tw != 0)) continue;
          if (tw * stride > 256) break;
          int th = 128 / tw;
          if (!halo && th > Ho) th = Ho;
          if (single_row_tiles) th = 1;                 // every output row has its own B operand
          if (MT == 2 && (tw * th) % 8 != 0) continue;
          const int box_rows = halo ? MT * th + 2 : MT * th * stride;
          if (box_rows > 256) continue;
          const long long tiles = static_cast<long long>(N) * ((Wo + tw - 1) / tw) * ((Ho + MT * th - 1) / (MT * th)) * nt;
          const int st_bytes = staging_for(staged, MT, BN);
          const RingCfg rc = ring_cfg(halo, kx_major, MT, tw, th, BN, kOperandBytes - st_bytes);
          // the MMA warps hold the slots of one wgmma group while they wait for the next group's
          if (rc.a_slots < (halo && !kx_major ? 3 : 2) || rc.b_slots < (halo ? 4 : 2)) continue;
          const double groups = static_cast<double>(taps) * kb_per_tap;   // one wgmma group per (tap, k-block)
          const double mma = static_cast<double>(MT) * taps * ksteps_tap * (30.0 + 0.25 * BN) + groups * 200.0;
          const double a_bytes = halo ? static_cast<double>(tw) * (MT * th + 2) * 128.0 * 3 * kb_per_tap
                                      : static_cast<double>(tw) * th * MT * 128.0 * taps * kb_per_tap;
          const double b_bytes = static_cast<double>(BN) * 128.0 * taps * kb_per_tap;
          const double l2 = (a_bytes + b_bytes) / 100.0;
          const double epi = MT * ((BN + 31) / 32) * (st_bytes > 0 ? kEpiStagedUnit : 500.0);
          // the epilogue does not overlap the main loop of the same warps: the two add up
          const double t = std::max(mma, l2) + epi + 800.0;
          double cost = static_cast<double>((tiles + sms - 1) / sms) * t;
          // 3x3 stride-1 convs, bf16, 32 images (scripts/conv_decompose.py, H100 SXM 700 W): halo mode is 7-38 % faster
          // than per-tap A loads when the channels end in a 32-byte tail group (Cin 196) or BN = 200; at Cin 128 / BN 128
          // and Cin 256 / BN 256 the two are within 4 % of each other. The model ranks them within a few percent either
          // way, so halo mode is preferred where it measurably wins.
          if (can_halo && f_halo < 0 && halo != ((tail32 || BN == 200) ? 1 : 0)) cost *= 1.25;
          if (cost < best.cost * (1.0 - 1e-9) || (cost < best.cost * (1.0 + 1e-9) && tw > best.TW)) {
            best = TileCfg{tw, th, MT, BN, nt, halo, cost};
          }
        }
      }
    }
  }
  }
  if (getenv("MFR_CONV_DEBUG"))
    fprintf(stderr, "[conv_gemm cfg] N%d %dx%d Cout%d R%d s%d kb%d -> TW%d TH%d MT%d BN%d nt%d halo%d cost %.0f\n", N, Ho, Wo,
            Cout, R, stride, kb_per_tap, best.TW, best.TH, best.MT, best.BN, best.n_tiles, best.halo, best.cost);
  return best;
}

}  // namespace

int conv_gemm_num_sms() { return sm_count(); }

int conv_gemm_build(const ConvGemmDesc& d, ConvGemmParams* p) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    fprintf(stderr, "[mfr_b200] cuTensorMapEncodeTiled unavailable (no CUDA driver?)\n");
    return MFR_ERR_CUDA;
  }
  const int es = d.in_bf16 ? 2 : 4;           // operand element size
  const int kblk = 128 / es;                  // K elements per 128-byte k-block
  const long long ldw_e = d.ldw > 0 ? d.ldw : d.Cin;
  if ((d.ldx * es) % 16 != 0 || (ldw_e * es) % 16 != 0 || (reinterpret_cast<uintptr_t>(d.x) & 15) ||
      (reinterpret_cast<uintptr_t>(d.w) & 15)) {
    fprintf(stderr, "[mfr_b200] conv_gemm: operand row strides must be multiples of 16 bytes, pointers 16B aligned\n");
    return MFR_ERR_ARG;
  }
  if (d.out_bf16 && ((d.Cout & 3) || (d.ldo & 3))) return MFR_ERR_ARG;   // bf16 output: vector path only
  if (d.stride != 1 && d.stride != 2) return MFR_ERR_ARG;
  memset(p, 0, sizeof(*p));
  p->N = d.N;
  p->Ho = (d.H + 2 * d.pad - d.R) / d.stride + 1;
  p->Wo = (d.W + 2 * d.pad - d.S) / d.stride + 1;
  p->Cout = d.Cout;
  p->Cin = d.Cin;
  p->R = d.R; p->S = d.S; p->stride = d.stride; p->pad = d.pad;
  p->kb_per_tap = (d.Cin + kblk - 1) / kblk;
  p->kblk = kblk;
  {  // MMAs in the last k-block of a tap: the channel tail is zero-filled by TMA, no need to multiply all of it
    const int tail = d.Cin - (p->kb_per_tap - 1) * kblk;
    const int ummak = kblk / 4;
    p->ksteps_last = (tail + ummak - 1) / ummak;
    // a tail of one k-step (<= 32 bytes of channels) is moved as 32-byte-wide tiles (32B swizzle) instead of zero-filled
    // 128-byte ones: Cin = 196 otherwise spends a quarter of its operand traffic on 4 channels
    p->tail32 = (p->ksteps_last == 1 && tail * es <= 32 && p->kb_per_tap > 1 && d.b_batched != 2) ? 1 : 0;
  }
  // Order of the fp32 sums over the taps, fixed per shape and the same in halo and per-tap mode, so that the tiling
  // never changes the result bits: kx-major for 3x3 stride-1 convs with at most 128 output channels, ky-major
  // otherwise (the orders the engine's convs have been summed in since halo mode exists)
  p->kx_major = (d.R == 3 && d.S == 3 && d.stride == 1 && d.pad == 1 && d.Cout <= 128) ? 1 : 0;
  p->act = d.act;
  p->act_cols = (d.act_cols > 0 && d.act != ACT_NONE) ? d.act_cols : d.Cout;   // without an activation act_cols is moot
  p->dyn_w = d.dyn_w;
  if (d.dyn_w != nullptr && (d.H != 1 || d.R != 1 || d.S != 1 || d.stride != 1)) return MFR_ERR_ARG;
  p->alpha = d.alpha;
  p->bias = d.bias;
  p->residual = d.residual;
  p->ldr = d.ldr;
  p->out = d.out;
  p->ldo = d.ldo;
  p->out_y_stride = d.out_y_stride > 0 ? d.out_y_stride : static_cast<long long>(p->Wo) * d.ldo;
  p->out_img_stride = d.out_img_stride > 0 ? d.out_img_stride : static_cast<long long>(p->Ho) * p->Wo * d.ldo;
  p->b_xor = d.b_xor;
  p->res_img_stride = static_cast<long long>(p->Ho) * p->Wo * d.ldr;
  // compile-time epilogue kind with TMA stores: a kind with an instantiation for the operand type (the N tile is
  // checked once it is chosen), every column activated, no residual together with a device row count, one B operand
  // per image at most, and output / residual rows that tensor maps can address (16-byte strides and pointers)
  p->epi = kEpiAny;
  {
    const int osz = d.out_bf16 ? 2 : 4;
    auto a16 = [](long long bytes) { return bytes % 16 == 0; };
    const int kind = epi_kind(d.out_bf16 != 0, d.residual != nullptr, d.act);
    if (staged_inst(kind, kMaxBN, d.in_bf16 != 0) && (d.dyn_w == nullptr || d.residual == nullptr) && d.b_batched != 2 &&
        p->act_cols >= p->Cout &&
        epilogue_vec2(*p) && (reinterpret_cast<uintptr_t>(d.bias) & 7) == 0 && (reinterpret_cast<uintptr_t>(d.out) & 15) == 0 &&
        a16(p->ldo * osz) && a16(p->out_y_stride * osz) && a16(p->out_img_stride * osz) &&
        (d.residual == nullptr || ((reinterpret_cast<uintptr_t>(d.residual) & 15) == 0 && a16(p->ldr * osz))))
      p->epi = kind;
  }
  const TileCfg cfg = choose_cfg(d.N, p->Ho, p->Wo, d.Cout, d.R, d.S, d.stride, d.pad, p->kb_per_tap, p->tail32 != 0,
                                 p->kx_major != 0, d.dyn_w == nullptr && d.b_batched != 2, d.b_batched == 2,
                                 p->epi == kEpiAny ? -1 : (d.out_bf16 ? 1 : 0));
  p->TW = cfg.TW; p->TH = cfg.TH; p->MT = cfg.MT; p->halo = cfg.halo;
  p->BN = cfg.BN; p->n_tiles = cfg.n_tiles;
  p->nt_fast = (!p->halo && p->n_tiles > 1) ? 1 : 0;
  p->tiles_x = (p->Wo + p->TW - 1) / p->TW;
  p->tiles_y = (p->Ho + p->MT * p->TH - 1) / (p->MT * p->TH);
  p->in_bf16 = d.in_bf16;
  p->out_bf16 = d.out_bf16;
  p->b_batched = d.b_batched;
  const int a_rows = p->halo ? p->MT * p->TH + 2 : p->MT * p->TH;   // pixel rows of the A box
  p->a_bytes = p->TW * a_rows * 128;
  p->b_bytes = p->BN * 128;                                           // multiple of 1 KB (BN % 8 == 0)
  // the narrow N tiles run the run-time generic epilogue: from here on p->epi names an instantiation
  if (p->epi != kEpiAny && !staged_inst(p->epi, p->BN, d.in_bf16 != 0)) p->epi = kEpiAny;
  if (p->epi != kEpiAny) {   // output / residual: {Cout, Wo, Ho, N}; the bounds clip ragged tiles and channels >= Cout
    const int osz = d.out_bf16 ? 2 : 4, cw = stage_cw(d.out_bf16 != 0);
    const CUtensorMapDataType dt = d.out_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    // TMA stores write whole 16-byte groups: the output map ends at the last full group, the rest goes from registers
    p->cout_tma = d.Cout / (16 / osz) * (16 / osz);
    cuuint64_t dims[4] = {(cuuint64_t)p->cout_tma, (cuuint64_t)p->Wo, (cuuint64_t)p->Ho, (cuuint64_t)d.N};
    cuuint32_t box[4] = {(cuuint32_t)cw, (cuuint32_t)p->TW, (cuuint32_t)p->TH, 1};
    cuuint32_t box2[4] = {(cuuint32_t)(p->BN % cw), (cuuint32_t)p->TW, (cuuint32_t)p->TH, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    auto encode = [&](CUtensorMap* tm, CUtensorMap* tm2, const float* ptr, long long ld, long long y_stride, long long img_stride) {
      cuuint64_t strides[3] = {(cuuint64_t)(ld * osz), (cuuint64_t)(y_stride * osz), (cuuint64_t)(img_stride * osz)};
      CUresult r = enc(tm, dt, 4, const_cast<float*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r == CUDA_SUCCESS && box2[0] > 0)
        r = enc(tm2, dt, 4, const_cast<float*>(ptr), dims, strides, box2, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      return r == CUDA_SUCCESS;
    };
    bool ok = encode(&p->tmO, &p->tmO2, d.out, p->ldo, p->out_y_stride, p->out_img_stride);
    dims[0] = d.Cout;   // the residual is read up to Cout (channels beyond come back as zeros)
    if (ok && d.residual != nullptr)
      ok = encode(&p->tmR, &p->tmR2, d.residual, p->ldr, static_cast<long long>(p->Wo) * p->ldr, p->res_img_stride);
    if (!ok) p->epi = kEpiAny;   // strides a tensor map cannot take: the run-time generic epilogue
  }
  // the staging buffer and the rings follow the final p->epi
  p->stage_bytes = staging_for(p->epi == kEpiAny ? -1 : (d.out_bf16 ? 1 : 0), p->MT, p->BN);
  {
    const RingCfg rc = ring_cfg(p->halo, p->kx_major != 0, p->MT, p->TW, p->TH, p->BN, kOperandBytes - p->stage_bytes);
    p->a_slot_bytes = rc.a_slot_bytes; p->a_slots = rc.a_slots; p->b_slots = rc.b_slots;
  }
  if (p->a_slots < (p->halo && !p->kx_major ? 3 : 2) || p->b_slots < (p->halo ? 4 : 2)) return MFR_ERR_ARG;

  {  // activations: {C, W, H, N}
    cuuint64_t dims[4] = {(cuuint64_t)d.Cin, (cuuint64_t)d.W, (cuuint64_t)d.H, (cuuint64_t)d.N};
    cuuint64_t strides[3] = {(cuuint64_t)d.ldx * es, d.x_y_stride > 0 ? (cuuint64_t)d.x_y_stride * es : (cuuint64_t)d.ldx * es * d.W,
                             d.x_img_stride > 0 ? (cuuint64_t)d.x_img_stride * es : (cuuint64_t)d.ldx * es * d.W * d.H};
    cuuint32_t box[4] = {(cuuint32_t)kblk, (cuuint32_t)(p->TW * d.stride),
                         (cuuint32_t)(p->halo ? p->MT * p->TH + 2 : p->MT * p->TH * d.stride), 1};
    cuuint32_t estr[4] = {1, (cuuint32_t)d.stride, (cuuint32_t)d.stride, 1};
    p->a_yx = 0;
    if (d.x_y_stride > 0 && d.x_y_stride < d.ldx) {   // rows interleaved inside a pixel: tensor-map strides must not decrease
      if (p->halo || d.stride != 1 || p->tail32) return MFR_ERR_ARG;
      p->a_yx = 1;
      std::swap(dims[1], dims[2]); std::swap(strides[0], strides[1]); std::swap(box[1], box[2]);
    }
    CUresult r = enc(&p->tmA, d.in_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
                     const_cast<float*>(d.x), dims,
                     strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      fprintf(stderr, "[mfr_b200] cuTensorMapEncodeTiled(A) failed: %d\n", (int)r);
      return MFR_ERR_CUDA;
    }
    if (p->tail32) {
      box[0] = static_cast<cuuint32_t>(32 / es);
      p->a_bytes2 = p->a_bytes / 4;
      r = enc(&p->tmA2, d.in_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
              const_cast<float*>(d.x), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) p->tail32 = 0;
    }
  }
  {  // weights: {Cin, Z, Cout}; Z = tap (shared weights) or image (batched B operand)
    const int taps = d.R * d.S;
    cuuint64_t dims[3];
    cuuint64_t strides[2];
    if (d.b_batched == 2) {   // per-(image, row) B operand: rank-4 map {Cin, Cout rows, y, image}
      cuuint64_t dims4[4] = {(cuuint64_t)d.Cin, (cuuint64_t)d.Cout, (cuuint64_t)p->Ho, (cuuint64_t)d.N};
      cuuint64_t strides4[3] = {(cuuint64_t)ldw_e * es, (cuuint64_t)d.w_y_stride * es, (cuuint64_t)d.w_img_stride * es};
      cuuint32_t box4[4] = {(cuuint32_t)kblk, (cuuint32_t)p->BN, 1, 1};
      cuuint32_t estr4[4] = {1, 1, 1, 1};
      p->b_yx = 0;
      if (d.w_y_stride < ldw_e) {
        p->b_yx = 1;
        std::swap(dims4[1], dims4[2]); std::swap(strides4[0], strides4[1]); std::swap(box4[1], box4[2]);
      }
      if (d.w_y_stride <= 0 || d.w_img_stride <= 0 || p->TH != 1 || p->MT != 1) return MFR_ERR_ARG;
      CUresult r4 = enc(&p->tmB, d.in_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
                        const_cast<float*>(d.w), dims4, strides4, box4, estr4, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r4 != CUDA_SUCCESS) {
        fprintf(stderr, "[mfr_b200] cuTensorMapEncodeTiled(B, per-row) failed: %d\n", (int)r4);
        return MFR_ERR_CUDA;
      }
      return MFR_OK;
    }
    if (d.b_batched) {
      const long long ldw = ldw_e;
      dims[0] = d.Cin; dims[1] = d.N; dims[2] = d.Cout;
      strides[0] = d.w_img_stride > 0 ? (cuuint64_t)d.w_img_stride * es : (cuuint64_t)d.Cout * ldw * es;  // next image
      strides[1] = (cuuint64_t)ldw * es;           // next output row
    } else {
      dims[0] = d.Cin; dims[1] = taps; dims[2] = d.Cout;
      strides[0] = (cuuint64_t)ldw_e * es;
      strides[1] = (cuuint64_t)ldw_e * es * taps;
    }
    cuuint32_t box[3] = {(cuuint32_t)kblk, 1, (cuuint32_t)p->BN};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(&p->tmB, d.in_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
                     const_cast<float*>(d.w), dims,
                     strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      fprintf(stderr, "[mfr_b200] cuTensorMapEncodeTiled(B) failed: %d\n", (int)r);
      return MFR_ERR_CUDA;
    }
    if (p->tail32) {
      box[0] = static_cast<cuuint32_t>(32 / es);
      p->b_bytes2 = p->b_bytes / 4;
      r = enc(&p->tmB2, d.in_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3,
              const_cast<float*>(d.w), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) {
        fprintf(stderr, "[mfr_b200] cuTensorMapEncodeTiled(B tail) failed: %d\n", (int)r);
        return MFR_ERR_CUDA;   // tmA2 exists already: both or neither
      }
    }
  }
  return MFR_OK;
}

namespace {
template <int BN_T, int MT_T, bool BF16, int EPI>
int launch_one(const ConvGemmParams& p, int grid, cudaStream_t stream) {
  static bool attr_seen[64] = {};
  if (first_call_on_device(attr_seen))
    MFR_CUDA_CHECK(cudaFuncSetAttribute(conv_gemm_kernel<BN_T, MT_T, BF16, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  conv_gemm_kernel<BN_T, MT_T, BF16, EPI><<<grid, kThreads, kSmemBytes, stream>>>(p);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
template <int BN_T, int MT_T, bool BF16>
int launch_typed(const ConvGemmParams& p, int grid, cudaStream_t stream) {
  if (p.epi == kEpiAny) return launch_one<BN_T, MT_T, BF16, kEpiAny>(p, grid, stream);
  if constexpr (BN_T >= 128) {   // the compile-time epilogue kinds (TMA stores) have their own instantiations
    switch (p.epi) {
      case kF32: return launch_one<BN_T, MT_T, BF16, kF32>(p, grid, stream);
      case kBf: if constexpr (BF16) return launch_one<BN_T, MT_T, true, kBf>(p, grid, stream); break;
      case kBfRelu: if constexpr (BF16) return launch_one<BN_T, MT_T, true, kBfRelu>(p, grid, stream); break;
      case kBfLeaky: if constexpr (BF16) return launch_one<BN_T, MT_T, true, kBfLeaky>(p, grid, stream); break;
      case kBfResRelu: if constexpr (BF16) return launch_one<BN_T, MT_T, true, kBfResRelu>(p, grid, stream); break;
    }
  }
  // conv_gemm_build names only kinds with an instantiation (staged_inst): a params block that gets here is not its own
  fprintf(stderr, "[mfr_b200] conv_gemm: no TMA-store kernel for epilogue kind %d at BN %d (%s operands)\n", p.epi, BN_T,
          BF16 ? "bf16" : "tf32");
  return MFR_ERR_UNSUPPORTED;
}
template <int BN_T, int MT_T>
int launch_inst(const ConvGemmParams& p, int grid, cudaStream_t stream) {
  return p.in_bf16 ? launch_typed<BN_T, MT_T, true>(p, grid, stream) : launch_typed<BN_T, MT_T, false>(p, grid, stream);
}
}  // namespace

int conv_gemm_launch(const ConvGemmParams& p, cudaStream_t stream) {
  const int total = p.N * p.tiles_y * p.tiles_x * p.n_tiles;
  if (total <= 0) return MFR_OK;
  const int grid = std::min(total, p.grid_limit > 0 ? std::min(p.grid_limit, conv_gemm_num_sms()) : conv_gemm_num_sms());
  if (p.MT == 2) {
    switch (p.BN) {
      case 32: return launch_inst<32, 2>(p, grid, stream);
      case 64: return launch_inst<64, 2>(p, grid, stream);
      case 128: return launch_inst<128, 2>(p, grid, stream);
    }
  } else if (p.MT == 1) {
    switch (p.BN) {
      case 32: return launch_inst<32, 1>(p, grid, stream);
      case 64: return launch_inst<64, 1>(p, grid, stream);
      case 128: return launch_inst<128, 1>(p, grid, stream);
      case 200: return launch_inst<200, 1>(p, grid, stream);
      case 256: return launch_inst<256, 1>(p, grid, stream);
    }
  }
  fprintf(stderr, "[mfr_b200] conv_gemm: no kernel for BN %d MT %d\n", p.BN, p.MT);
  return MFR_ERR_UNSUPPORTED;
}

float conv_gemm_time_prebuilt(const ConvGemmParams& p, int iters, cudaStream_t st) {
  if (getenv("MFR_CONV_DEBUG"))
    fprintf(stderr, "[conv_gemm cfg] TW%d TH%d MT%d BN%d nt%d halo%d slots %d/%d\n", p.TW, p.TH, p.MT, p.BN, p.n_tiles, p.halo,
            p.a_slots, p.b_slots);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  for (int i = 0; i < 5; ++i) conv_gemm_launch(p, st);
  cudaEventRecord(e0, st);
  for (int i = 0; i < iters; ++i) conv_gemm_launch(p, st);
  cudaEventRecord(e1, st);
  cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return ms * 1000.f / iters;
}

}  // namespace mfr
