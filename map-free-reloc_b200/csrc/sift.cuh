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

struct SiftPairs;
int sift_pairs_create(int P, int H, int W, int nfeatures, int max_candidates, int root_sift, float ratio, SiftPairs** out);
void sift_pairs_destroy(SiftPairs* e);
EngineCore& engine_core(SiftPairs* e);
int sift_forward_pairs(SiftPairs* e, const unsigned char* img0, const unsigned char* img1, cudaStream_t st);
int sift_pairs_set_map(SiftPairs* e, const unsigned char* img0, cudaStream_t st);
int sift_forward_shared(SiftPairs* e, const unsigned char* img1, cudaStream_t st);
void sift_pair_outputs(SiftPairs* e, mfr_sift_pair_outputs* o);

}  // namespace mfr
