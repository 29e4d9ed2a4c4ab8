// Pose back end (see geometry.cu).
#pragma once
#include "common.cuh"

namespace mfr {

struct PoseSolver;

int pose_solver_create(int max_pairs, int max_pts, int max_hyp, PoseSolver** out);
void pose_solver_destroy(PoseSolver* s);
double* pose_solver_Rd(PoseSolver* s);
double* pose_solver_td(PoseSolver* s);
// named scratch buffer of the handle (see mfr_pose_solver_debug_tensor); words = its size in 4-byte words
int pose_solver_debug_tensor(PoseSolver* s, const char* name, void** ptr, long long* words);

int emat_ransac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                const float* K0, const float* K1, float pix_thr, int num_hyp, unsigned long long seed,
                int lo_enabled, float* R, float* t, int* n_inl, unsigned char* mask, cudaStream_t st);
// the same solve repeated at h0, min(max_hyp, 4 h0), ... for the pairs whose CONFIDENCE stopping rule asks for more
// (mfr_emat_ransac_escalate); budgets_out: device int[P] or nullptr
int emat_ransac_escalate(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                         const float* K0, const float* K1, float pix_thr, int num_hyp, unsigned long long seed,
                         int lo_enabled, float* R, float* t, int* n_inl, unsigned char* mask, double confidence,
                         int max_hyp, int* budgets_out, cudaStream_t st);
// emat_ransac_escalate with MAGSAC++ scoring and sigma-consensus++ in place of MSAC and its LO (mfr_emat_magsac)
int emat_magsac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P, const float* K0,
                const float* K1, float pix_thr, int num_hyp, unsigned long long seed, float* R, float* t, int* n_inl,
                unsigned char* mask, double confidence, int max_hyp, int* budgets_out, cudaStream_t st);
int scale_from_depth(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                     const float* K0, const float* K1, const unsigned char* mask, const double* Rd,
                     const double* td, const float* depth0, const float* depth1, int H, int W,
                     float scale_thr, float* R_out, float* t_out, int* inliers, cudaStream_t st);
int pnp_ransac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
               const float* K0, const float* K1, const float* depth0, int H, int W, int num_hyp,
               float reproj_thr, unsigned long long seed, float* R, float* t, int* n_inl,
               unsigned char* mask, cudaStream_t st);
int pnp_ransac_escalate(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                        const float* K0, const float* K1, const float* depth0, int H, int W, int num_hyp,
                        float reproj_thr, unsigned long long seed, float* R, float* t, int* n_inl,
                        unsigned char* mask, double confidence, int max_hyp, int* budgets_out, cudaStream_t st);

int procrustes_ransac(PoseSolver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                      const float* K0, const float* K1, const float* depth0, const float* depth1, int H, int W,
                      int num_hyp, float max_corr_dist, unsigned long long seed, float* R, float* t, int* n_inl,
                      cudaStream_t st);

// ICP refinement over the full depth clouds (pose_solver.py:289-315), starting from (R_in, t_in) [P][9] / [P][3] (NaN = skip)
int icp_refine(PoseSolver* s, const float* depth0, const float* depth1, int H, int W, int P, const float* K0, const float* K1,
               const float* R_in, const float* t_in, float max_corr_dist, int max_iter, float rel_fitness, float rel_rmse,
               float* R, float* t, int* n_inl, cudaStream_t st);

}  // namespace mfr
