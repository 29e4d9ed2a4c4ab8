// SuperPoint + SuperGlue matcher engine (see spsg_engine.cu).
#pragma once
#include "common.cuh"

namespace mfr {

struct EngineCore;
struct SpsgEngine;

int spsg_create(int B, int H, int W, int max_kp, int nms_radius, float kp_thr, int border, int sinkhorn_iters,
                float match_thr, int precision, SpsgEngine** out);
void spsg_destroy(SpsgEngine* e);
EngineCore& engine_core(SpsgEngine* e);
int spsg_forward(SpsgEngine* e, const float* img0, const float* img1, cudaStream_t st);
int spsg_set_map(SpsgEngine* e, const float* img0, cudaStream_t st);
int spsg_forward_shared(SpsgEngine* e, const float* img1, cudaStream_t st);
void spsg_outputs(SpsgEngine* e, mfr_spsg_outputs* o);
int spsg_forward_superglue(SpsgEngine* e, const int* counts, const float* kpts, const float* scores, const float* desc,
                           cudaStream_t st);

}  // namespace mfr
