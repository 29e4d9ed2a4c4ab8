// SuperPoint + SuperGlue matcher engine (see spsg_engine.cu).
#pragma once
#include "common.cuh"

namespace mfr {

struct SpsgEngine;

struct SpsgOutputs {
  const int* counts;          // [2B] keypoints per image, pair-interleaved (2p = image0 of pair p)
  const float* keypoints;     // [2B][K][2] pixel (x, y)
  const float* scores;        // [2B][K]
  const float* descriptors;   // [2B][K][desc_ld] SuperPoint descriptors (token major)
  int desc_ld;
  const int* matches0;        // [B][K]  index into image1's keypoints or -1
  const float* matching_scores0;  // [B][K]
  const int* m_offsets;       // [B+1] offsets into mkpts0/mkpts1
  const float* mkpts0; const float* mkpts1;   // [total][2] matched coordinates, ordered by (pair, i)
  int max_keypoints;
};

int spsg_create(int B, int H, int W, int max_kp, int nms_radius, float kp_thr, int border, int sinkhorn_iters,
                float match_thr, int precision, SpsgEngine** out);
void spsg_destroy(SpsgEngine* e);
int spsg_num_weights(const SpsgEngine* e);
const char* spsg_weight_name(const SpsgEngine* e, int i);
long long spsg_weight_numel(const SpsgEngine* e, int i);
int spsg_set_weight(SpsgEngine* e, int i, const float* host, long long numel, cudaStream_t st);
int spsg_forward(SpsgEngine* e, const float* img0, const float* img1, cudaStream_t st);
int spsg_set_map(SpsgEngine* e, const float* img0, cudaStream_t st);
int spsg_forward_shared(SpsgEngine* e, const float* img1, cudaStream_t st);
void spsg_set_graph(SpsgEngine* e, int on);
SpsgOutputs spsg_outputs(SpsgEngine* e);
int spsg_debug_tensor(SpsgEngine* e, const char* name, float** ptr, long long* numel);
int spsg_num_launches(const SpsgEngine* e);
int spsg_forward_superglue(SpsgEngine* e, const int* counts, const float* kpts, const float* scores, const float* desc,
                           cudaStream_t st);

}  // namespace mfr
