#pragma once
#include "common.cuh"
namespace mfr {
int knn2_l2(const float* q, int nq, const float* t, int nt, int dim, int* idx1, float* dist1, int* idx2,
            float* dist2, cudaStream_t st);
// 2-NN of image 2p's rows among image 2p+1's, for P pairs of a pair-interleaved [2P][cap][dim] descriptor array;
// row counts are read from counts[2P] on the device. Outputs [P][cap].
int knn2_l2_pairs(const float* desc, const int* counts, int P, int cap, int dim, int* idx1, float* dist1, int* idx2,
                  float* dist2, cudaStream_t st);
// 2-NN of one query set q [cap][dim] (q_count[0] rows, shared by every pair) among each train set p of t [P][cap][dim]
// (t_counts[p] rows); counts are read on the device. Outputs [P][cap].
int knn2_l2_shared(const float* q, const int* q_count, const float* t, const int* t_counts, int P, int cap, int dim,
                   int* idx1, float* dist1, int* idx2, float* dist2, cudaStream_t st);
}
