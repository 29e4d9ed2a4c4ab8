// LoFTR matcher engine (see loftr_engine.cu).
#pragma once
#include "common.cuh"

namespace mfr {

struct EngineCore;
struct LoftrEngine;

int loftr_create(int B, int H, int W, float thr, int border, float temperature, int precision, int reserved_sms,
                 LoftrEngine** out);
void loftr_destroy(LoftrEngine* e);
EngineCore& engine_core(LoftrEngine* e);
int loftr_forward(LoftrEngine* e, const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st);
int loftr_set_map(LoftrEngine* e, const float* img0, int src_h, int src_w, cudaStream_t st);
int loftr_forward_shared(LoftrEngine* e, const float* img1, int src_h, int src_w, cudaStream_t st);
void loftr_outputs(LoftrEngine* e, mfr_loftr_outputs* o);
int loftr_profile(LoftrEngine* e, const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st,
                  int max_steps, float* ms, double* flops, int* kinds, char* names);
int loftr_run_steps(LoftrEngine* e, int begin, int end, cudaStream_t st);

}  // namespace mfr
