// SIFT detector + descriptor engine (see sift.cu).
#pragma once
#include "common.cuh"

namespace mfr {

struct SiftEngine;

struct SiftOutputs {
  const int* counts;          // [B] keypoints per image after selection
  const int* raw_counts;      // [B] oriented keypoints before selection (true count, may exceed capacity)
  const int* extrema_counts;  // [B] refined extrema before orientation (true count, may exceed capacity)
  const float* keypoints;     // [B][cap][5] x, y, size, angle, response (input pixels, OpenCV's KeyPoint fields)
  const int* octaves;         // [B][cap] OpenCV's packed KeyPoint::octave
  const float* descriptors;   // [B][cap][128] SIFT (integer-valued) or RootSIFT rows
  int capacity;
};

int sift_create(int B, int H, int W, int nfeatures, int max_candidates, int root_sift, SiftEngine** out);
void sift_destroy(SiftEngine* e);
int sift_detect(SiftEngine* e, const unsigned char* imgs, cudaStream_t st);
void sift_set_graph(SiftEngine* e, int on);
SiftOutputs sift_outputs(SiftEngine* e);
int sift_match_pairs(SiftEngine* e, float ratio, float* kpts0, float* kpts1, int* offsets, cudaStream_t st);
int sift_debug_tensor(SiftEngine* e, const char* name, float** ptr, long long* numel);
int sift_profile(SiftEngine* e, const unsigned char* imgs, float* ms, cudaStream_t st);

}  // namespace mfr
