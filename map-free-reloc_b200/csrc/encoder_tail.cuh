// Fused tail of one LoFTREncoderLayer (etc/feature_matching_baselines/LoFTR/src/loftr/loftr_module/transformer.py:52-58):
//   message = norm1(merge(message));  message = mlp(cat([x, message]));  x = x + norm2(message)
// as ONE persistent wgmma kernel per layer call (bf16 engine mode). See encoder_tail.cu.
#pragma once
#include "common.cuh"

namespace mfr {

struct alignas(64) EncoderTailParams {
  CUtensorMap tmMsg;  // bf16 [rows][C]  attention message (row stride ld_msg)      box {64, 128}
  CUtensorMap tmX;    // bf16 [rows][C]  x half of the token shadow (row stride ld_xb) box {64, 128}
  CUtensorMap tmWm;   // bf16 [C][C]     merge.weight                                 box {64, 128}
  CUtensorMap tmW0;   // bf16 [2C][2C]   mlp.0.weight                                 box {64, 64 (C = 256) | 128}
  CUtensorMap tmW2;   // bf16 [C][2C]    mlp.2.weight                                 box {64, 128}
  const float *g1, *b1, *g2, *b2;   // norm1 / norm2 affine parameters [C]
  float* x;            // fp32 residual stream, in/out, row stride ldx (elements)
  unsigned short* xb;  // bf16 shadow of x, out, row stride ld_xb (elements)
  long long ldx, ld_xb;
  int C;               // 256 (coarse level) or 128 (fine level)
  int n_img;           // row blocks ("images" / window sides), each rows_cap rows apart
  long long rows_cap;  // rows per block (capacity)
  const int* dyn_rows; // device: live rows per block (null = rows_cap)
};

struct EncoderTailDesc {
  const void* msg; long long ld_msg;      // bf16
  const void* xb_in; long long ld_xb;     // bf16 shadow (x half is read, and rewritten with the layer's output)
  const void *w_merge, *w_mlp0, *w_mlp2;  // bf16, row-major [out][in]
  const float *g1, *b1, *g2, *b2;
  float* x; long long ldx;
  int C, n_img; long long rows_cap; const int* dyn_rows;
};

int encoder_tail_build(const EncoderTailDesc& d, EncoderTailParams* p);
int encoder_tail_launch(const EncoderTailParams& p, cudaStream_t st);

}  // namespace mfr
