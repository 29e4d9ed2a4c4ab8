// LoFTR matcher engine (see loftr_engine.cu).
#pragma once
#include "common.cuh"

namespace mfr {

struct LoftrEngine;

struct LoftrOutputs {
  const int* m_total;     // [4] {M, 2M, 25M, 50M} total matches of the batch
  const int* m_offsets;   // [B+1] first match of every pair (matches are ordered by (pair, i))
  const int* b_ids; const int* i_ids; const int* j_ids;   // [capacity]
  const float* mconf;                                      // [capacity]
  const float* mkpts0_f; const float* mkpts1_f;            // [capacity][2] pixel (x, y)
  const float* mkpts1_c; const float* expec_f;             // [capacity][2], [capacity][3]
  int capacity;
};

int loftr_create(int B, int H, int W, float thr, int border, float temperature, int precision, int reserved_sms,
                 LoftrEngine** out);
void loftr_destroy(LoftrEngine* e);
int loftr_num_weights(const LoftrEngine* e);
const char* loftr_weight_name(const LoftrEngine* e, int i);
long long loftr_weight_numel(const LoftrEngine* e, int i);
int loftr_set_weight(LoftrEngine* e, int i, const float* host, long long numel, cudaStream_t st);
int loftr_forward(LoftrEngine* e, const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st);
int loftr_set_map(LoftrEngine* e, const float* img0, int src_h, int src_w, cudaStream_t st);
int loftr_forward_shared(LoftrEngine* e, const float* img1, int src_h, int src_w, cudaStream_t st);
void loftr_set_graph(LoftrEngine* e, int on);
LoftrOutputs loftr_outputs(LoftrEngine* e);
int loftr_debug_tensor(LoftrEngine* e, const char* name, float** ptr, long long* numel);
int loftr_num_steps(const LoftrEngine* e);
int loftr_num_launches(const LoftrEngine* e);
int loftr_profile(LoftrEngine* e, const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st,
                  int max_steps, float* ms, double* flops, int* kinds, char* names);

}  // namespace mfr
