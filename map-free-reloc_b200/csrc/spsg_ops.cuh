// SIMT kernels of the SuperPoint + SuperGlue matcher (launch wrappers). fp32 unless named bf16, channel-last.
#pragma once
#include "common.cuh"

namespace mfr {

int sp_conv1a(const float* img, const float* w /*[64][9]*/, const float* bias, float* out, int N, int H, int W,
              cudaStream_t st);
int maxpool2x2(const float* in, float* out, int N, int H, int W, int C, cudaStream_t st);
// bf16 variants of the engine's bf16 mode: conv1a with a bf16 output, 2x2 max-pool over bf16 (C % 8 == 0)
int sp_conv1a_bf16(const float* img, const float* w, const float* bias, void* out, int N, int H, int W, cudaStream_t st);
int maxpool2x2_bf16(const void* in, void* out, int N, int H, int W, int C, cudaStream_t st);
// softmax over 65 logits (row stride ldc), drop dustbin, depth-to-space -> scores [N][8h][8w]
int sp_score_map(const float* logits, int ldc, float* scores, int N, int h, int w, cudaStream_t st);
// simple_nms (superpoint.py:47-62): mask (0/1 floats); t0..t3 scratch of the same size
int sp_nms(const float* scores, float* mask, float* t0, float* t1, float* t2, float* t3, int N, int H, int W, int r,
           cudaStream_t st);
// threshold + border + top-k (superpoint.py:170-187) -> kpts [N][max_kp][2] (x,y), kscores, counts
int sp_select_keypoints(const float* scores, const float* mask, int N, int H, int W, float thr, int border,
                        int max_kp, float* kpts, float* kscores, int* counts, cudaStream_t st);
int l2norm256(float* x, size_t rows, cudaStream_t st);
int sp_sample_descriptors(const float* dense, const float* kpts, const int* counts, int N, int h, int w, int max_kp,
                          float* out, long long ldo, cudaStream_t st);
// shared map frame: pair-interleaved counts [2B], kpts [2B][K][2], scores [2B][K], desc [2B][K][256] with image 2b =
// the map's SuperPoint outputs (counts [1], kpts [K][2], ...) and image 2b + 1 = query b's (q_* [B][...])
int sp_pair_interleave(const int* map_counts, const float* map_kpts, const float* map_scores, const float* map_desc,
                       const int* q_counts, const float* q_kpts, const float* q_scores, const float* q_desc, int B, int max_kp,
                       int* counts, float* kpts, float* scores, float* desc, cudaStream_t st);
// SuperGlue
int sg_kenc_input(const float* kpts, const float* kscores, float* out, int total, int H, int W, cudaStream_t st);
// tensor-core attention helpers (see spsg_ops.cu): in-place row softmax of the [img][4][K][K] scores, V transpose
int sg_softmax_rows(float* S, const int* counts, int cross, int max_kp, int n_img, cudaStream_t st);
int sg_transpose_v(const float* qkv, long long ld, float* vt, int max_kp, int n_img, cudaStream_t st);
int sg_sinkhorn(const float* S, int ldS, const int* counts, float alpha, int iters, int max_kp, int n_pairs,
                float* u, float* v, cudaStream_t st);
int sg_extract_matches(const float* S, int ldS, const int* counts, const float* u, const float* v, float thr,
                       const float* kpts, int max_kp, float* rmax, int* rarg, int* carg, int* matches0,
                       float* mscores0, float* mk0, float* mk1, int* m_offsets, int n_pairs, cudaStream_t st);

}  // namespace mfr
