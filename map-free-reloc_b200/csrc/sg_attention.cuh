// SuperGlue multi-head softmax attention (superglue.py:85-89), bf16 engine mode, fused on wgmma:
//   msg[img][q][64 h + d] = sum_k softmax_k(Q_h[q] . K_h[k] / 8) V_h[k][d],   keys and values of image img ^ cross
// 4 heads of 64. qkv [n_img][max_kp][ldq] bf16 holds q | k | v (columns 0-255, 256-511, 512-767, head h at 64 h);
// msg [n_img][max_kp][ldo] bf16. Images attend over the counts[img ^ cross] keys of their partner; query rows at or past
// counts[img] get an all-zero message, and so does every row when the partner has no keypoint. The scores never leave
// the SM.
#pragma once
#include "common.cuh"

namespace mfr {

struct alignas(64) SgAttentionParams {
  CUtensorMap tm;             // qkv as {768 columns, max_kp rows, n_img}, box {64, 128, 1}, 128B swizzle, zero OOB fill
  const int* counts;
  unsigned short* msg;
  long long ldo;
  int n_img, max_kp, cross;
};

// max_kp: multiple of 16 in [16, 2048]; cross in {0, 1} (n_img even when 1); ldq >= 768 and ldo >= 256 in elements,
// qkv 16-byte and msg 4-byte aligned, row strides of 16 / 4 bytes
int sg_attention_build(const void* qkv, long long ldq, const int* counts, int n_img, int max_kp, int cross, void* msg,
                       long long ldo, SgAttentionParams* p);
int sg_attention_launch(const SgAttentionParams& p, cudaStream_t st);

}  // namespace mfr
