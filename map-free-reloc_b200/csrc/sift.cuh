// SIFT detector + descriptor engine (see sift.cu).
#pragma once
#include "common.cuh"

namespace mfr {

struct EngineCore;
struct SiftEngine;

int sift_create(int B, int H, int W, int nfeatures, int max_candidates, int root_sift, SiftEngine** out);
void sift_destroy(SiftEngine* e);
EngineCore& engine_core(SiftEngine* e);
int sift_detect(SiftEngine* e, const unsigned char* imgs, cudaStream_t st);
void sift_outputs(SiftEngine* e, mfr_sift_outputs* o);
int sift_match_pairs(SiftEngine* e, float ratio, float* kpts0, float* kpts1, int* offsets, cudaStream_t st);
int sift_profile(SiftEngine* e, const unsigned char* imgs, float* ms, cudaStream_t st);

}  // namespace mfr
