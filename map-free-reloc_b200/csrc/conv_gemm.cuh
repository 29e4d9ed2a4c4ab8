// Implicit-GEMM convolution / GEMM on the Hopper tensor cores (wgmma, TF32 or BF16 in, fp32 accumulate).
//
// One kernel serves every GEMM-shaped op of the matcher networks:
//   * 3x3 / 1x1 convolutions over NHWC activations (stride 1 or 2, zero padding),
//   * Linear layers over token sequences  (H = 1, W = tokens),
//   * batched  X * Y^T  products (correlation volumes), B operand indexed by the image.
// out[n, y, x, co] = act( alpha * sum_{ky,kx,ci} in[n, y*s-p+ky, x*s-p+kx, ci] * w[co, ky*S+kx, ci]
//                         + bias[co] + residual[n, y, x, co] )
#pragma once
#include "common.cuh"

namespace mfr {

enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY = 2, ACT_ELU1 = 3 };

struct alignas(64) ConvGemmParams {
  CUtensorMap tmA;  // rank 4 {C, W, H, N}   box {32|64, TW*s, MT*TH*s (halo: MT*TH+2), 1}, 128B swizzle, zero OOB fill
  CUtensorMap tmB;  // rank 3 {Cin, Z, Cout} box {32, 1, BN}          (Z = filter tap or image)
  CUtensorMap tmA2; // channel tail (tail32): same tensors, 32-byte-wide boxes, 32B swizzle — the last k-block of a tap then moves
  CUtensorMap tmB2; //   a quarter of the bytes (Cin = 196 leaves 4 channels for it) and issues one MMA per tap
  CUtensorMap tmO;  // TMA-store epilogue (epi >= 0): output rank 4 {Cout, Wo, Ho, N}, box {64 bf16 | 32 fp32, TW, TH, 1}, 128B swizzle
  CUtensorMap tmO2; //   the narrow last box of a BN = 200 tile: {BN % 64 | BN % 32 channels, TW, TH, 1}, no swizzle
  CUtensorMap tmR;  //   residual, same boxes as tmO / tmO2 (loaded into the staging buffer)
  CUtensorMap tmR2;
  int N, Ho, Wo, Cout, Cin;
  int R, S, stride, pad;
  int TW, TH, tiles_x, tiles_y;
  int BN, n_tiles, kb_per_tap, b_batched;   // BN: 32, 64, 128, 200 or 256 (the wgmma N)
  int a_bytes, b_bytes;   // TMA transaction bytes of one A / B load
  int MT;                 // 128-pixel sub-tiles per CTA tile (2 only when BN <= 128: the accumulators of a tile are registers)
  int halo;               // 3x3 stride-1 conv: A is loaded as a (MT*TH+2)-row box per (k-block, kx) and the three
                          // ky taps read it at row offsets 0, TW, 2*TW (TW % 8 == 0 keeps the swizzle phase)
  int kx_major;           // 3x3: the taps are summed column by column (kx outer, ky inner) instead of row by row
  int a_slots, b_slots;   // depth of the A ring / B ring (two rings: one A slot serves 3 B tiles in halo mode, each
                          // B tile is one wgmma group)
  int a_slot_bytes;
  int grid_limit;         // > 0: at most this many CTAs (the engine leaves SMs to the pose back end of the previous batch during the first layers)
  int nt_fast;            // work-item order: N tile index fastest (generic mode with several N tiles: the A tiles of a pixel tile stay in L2)
  int ksteps_last;        // MMAs issued for the last k-block of a tap (channel tail)
  int tail32;             // the tail fits one 32-byte k-step: it is loaded through tmA2 / tmB2 (a_bytes2 / b_bytes2 per load)
  int a_bytes2, b_bytes2;
  int act, act_cols;    // activation applies to output channels < act_cols
  int epi;              // epilogue kind with a compile-time body and TMA stores (conv_gemm.cu: epi_kind), -1: run-time
                        // generic epilogue
  int stage_bytes;      // shared-memory staging buffer of the TMA-store epilogue (0: none)
  int cout_tma;         // channels written by the TMA stores (Cout rounded down to 16 bytes; the rest from registers)
  int in_bf16, out_bf16;  // operands bf16 instead of fp32 (tf32 MMA); out/residual bf16
  int kblk;             // K elements per 128-byte k-block: 32 (fp32) or 64 (bf16)
  const int* dyn_w;     // optional device int: effective W (rows of a token GEMM), H must be 1
  float alpha;
  const float* bias;
  const float* residual;
  float* out;
  long long ldr, ldo;
  long long out_img_stride, res_img_stride;  // elements between images of out / residual
  long long out_y_stride;                    // elements between output rows (Wo * ldo when dense)
  int b_xor;
  int a_yx, b_yx;                            // tensor map dims 1 and 2 swapped (row stride smaller than the pixel / filter-row stride:
                                             // attention heads interleaved inside a token row) -> coordinate order (c, y, x|n, img)
};

// Describes one op; build once (tensor maps are encoded on the host), launch many times.
struct ConvGemmDesc {
  const float* x;      // activations, NHWC with pixel stride ldx (elements)
  int N, H, W, Cin;
  long long ldx;
  const float* w;      // [Cout][R*S][Cin] (Cin fastest); for batched GEMM: [N][Cout][ldw]
  int Cout, R, S, stride, pad;
  int b_batched;       // 0: shared weights; 1: per-image B operand; 2: per-(image, output row y) B operand (H = e.g. attention
                       //    heads): w[(img ^ b_xor)][y][Cout rows][Cin] with strides w_img_stride / w_y_stride / ldw
  long long ldw;       // row stride of w in elements (0 = Cin): per tap for shared weights, per row if batched
  int act_cols;        // 0 = all output channels
  const int* dyn_w;    // optional device row count (token GEMMs with data-dependent length)
  long long x_img_stride, w_img_stride, out_img_stride;  // elements between images; 0 = dense
  long long x_y_stride, w_y_stride, out_y_stride;        // elements between rows y of x / of w (b_batched 2) / of out; 0 = dense
  int b_xor;                                             // b_batched 2: the B operand of image i is taken from image i ^ b_xor
  int in_bf16, out_bf16;  // x / w are bf16 ; out / residual are bf16 (pointers reinterpret the storage)
  const float* bias;   // [Cout] or null
  const float* residual;  // NHWC like out (pixel stride ldr) or null
  long long ldr;
  int act;
  float alpha;
  float* out;          // NHWC, pixel stride ldo
  long long ldo;
};

int conv_gemm_build(const ConvGemmDesc& d, ConvGemmParams* p);
int conv_gemm_launch(const ConvGemmParams& p, cudaStream_t stream);
int conv_gemm_num_sms();
float conv_gemm_time_prebuilt(const ConvGemmParams& p, int iters, cudaStream_t st);

}  // namespace mfr
