// C ABI of libmfr_b200.so (declared in include/mfr_b200.h).
#include "../../include/mfr_b200.h"

#include <algorithm>
#include <cstdlib>
#include "common.cuh"
#include "conv_gemm.cuh"
#include "encoder_tail.cuh"
#include "engine_core.cuh"
#include "loftr_engine.cuh"
#include "loftr_ops.cuh"
#include "spsg_engine.cuh"
#include "sg_attention.cuh"
#include "geometry_solvers.cuh"
#include "geometry.cuh"
#include "descriptor_match.cuh"
#include "sift.cuh"

namespace mfr {   // image_io.cu
int resize_linear(const void* src, int src_is_u8, int sw, int sh, long long src_stride, int channels, float* dst, int dw, int dh,
                  int mode, float out_scale, int chw, cudaStream_t st);
int jpeg_info(const unsigned char* data, size_t length, int* width, int* height, int* components);
int jpeg_decode(const unsigned char* data, size_t length, int rgb, unsigned char* dst, int width, int height, cudaStream_t st);
struct JpegDecoder;
int jpeg_decoder_create(int max_images, long long max_bytes, long long max_pixels, JpegDecoder** out);
void jpeg_decoder_destroy(JpegDecoder* dec);
int jpeg_decode_batch(JpegDecoder* dec, const unsigned char* const* data, const long long* lengths, int n, int rgb,
                      unsigned char* const* dst, int* status, cudaStream_t st);
void jpeg_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* status);
int jpeg_host_decode(const unsigned char* data, size_t length, int rgb, unsigned char* dst, int width, int height);
struct PngDecoder;
int png_info(const unsigned char* data, size_t length, int* width, int* height, int* bit_depth);
int png_decoder_create(int max_images, long long max_bytes, long long max_pixels, PngDecoder** out);
void png_decoder_destroy(PngDecoder* dec);
void png_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* bit_depth,
                    int* status);
int png_decode_batch(PngDecoder* dec, const unsigned char* const* data, const long long* lengths, int n, int out_kind,
                     void* const* dst, int* status, cudaStream_t st);
int png_host_decode(const unsigned char* data, size_t length, int out_kind, void* dst, int width, int height);
int png_decoder_kernel_ms(PngDecoder* dec, float* ms);
}
struct mfr_jpeg_decoder {
  mfr::JpegDecoder* d;
};
struct mfr_png_decoder {
  mfr::PngDecoder* d;
};
namespace mfr {   // metrics.cu
int pose_metrics(const double* q_gt, const double* t_gt, const double* q_est, const double* t_est, const double* K, int W, int H,
                 int n, double* trans_err, double* rot_err, double* reproj_err, cudaStream_t st);
}

// The engine operations every engine shares (weight enumeration and upload, debug buffers, the graph switch, launch
// counts) act on its EngineCore.
template <class Handle>
static mfr::EngineCore& core(const Handle* h) { return mfr::engine_core(h->e); }

extern "C" {

int mfr_version(void) { return 101; }

int mfr_device_sm_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return 0;
  return mfr::conv_gemm_num_sms();
}

int mfr_conv2d_nhwc_tf32(const float* x, int N, int H, int W, int Cin, long long ldx,
                         const float* w, int Cout, int R, int S, int stride, int pad,
                         int b_batched, const float* bias, const float* residual, long long ldr,
                         int act, float alpha, float* out, long long ldo, void* stream) {
  mfr::ConvGemmDesc d{};
  d.x = x; d.N = N; d.H = H; d.W = W; d.Cin = Cin; d.ldx = ldx;
  d.w = w; d.Cout = Cout; d.R = R; d.S = S; d.stride = stride; d.pad = pad;
  d.b_batched = b_batched; d.bias = bias; d.residual = residual; d.ldr = ldr;
  d.act = act; d.alpha = alpha; d.out = out; d.ldo = ldo;
  mfr::ConvGemmParams p;
  int rc = mfr::conv_gemm_build(d, &p);
  if (rc != MFR_OK) return rc;
  return mfr::conv_gemm_launch(p, static_cast<cudaStream_t>(stream));
}

int mfr_conv2d_nhwc_bf16(const void* x, int N, int H, int W, int Cin, long long ldx, const void* w, long long ldw,
                         int Cout, int R, int S, int stride, int pad, const float* bias, const void* residual,
                         long long ldr, int act, float alpha, void* out, long long ldo, int out_bf16, void* stream) {
  mfr::ConvGemmDesc d{};
  d.x = static_cast<const float*>(x); d.N = N; d.H = H; d.W = W; d.Cin = Cin; d.ldx = ldx;
  d.w = static_cast<const float*>(w); d.ldw = ldw; d.Cout = Cout; d.R = R; d.S = S; d.stride = stride; d.pad = pad;
  d.bias = bias; d.residual = static_cast<const float*>(residual); d.ldr = ldr; d.act = act; d.alpha = alpha;
  d.out = static_cast<float*>(out); d.ldo = ldo; d.in_bf16 = 1; d.out_bf16 = out_bf16;
  mfr::ConvGemmParams p;
  int rc = mfr::conv_gemm_build(d, &p);
  if (rc != MFR_OK) return rc;
  return mfr::conv_gemm_launch(p, static_cast<cudaStream_t>(stream));
}

int mfr_token_gemm_dyn_rows(const void* x, int n_img, int rows_cap, int Cin, long long ldx, const void* w, long long ldw,
                            int in_bf16, int Cout, const float* bias, int act, void* out, long long ldo, int out_bf16,
                            const int* dyn_rows, void* stream) {
  if (dyn_rows == nullptr) return MFR_ERR_ARG;
  mfr::ConvGemmDesc d{};
  d.x = static_cast<const float*>(x); d.N = n_img; d.H = 1; d.W = rows_cap; d.Cin = Cin; d.ldx = ldx;
  d.w = static_cast<const float*>(w); d.ldw = ldw; d.Cout = Cout; d.R = 1; d.S = 1; d.stride = 1; d.pad = 0;
  d.bias = bias; d.act = act; d.alpha = 1.f; d.out = static_cast<float*>(out); d.ldo = ldo;
  d.in_bf16 = in_bf16; d.out_bf16 = out_bf16; d.dyn_w = dyn_rows;
  mfr::ConvGemmParams p;
  int rc = mfr::conv_gemm_build(d, &p);
  if (rc != MFR_OK) return rc;
  return mfr::conv_gemm_launch(p, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------ LoFTR
struct mfr_loftr { mfr::LoftrEngine* e; };

int mfr_loftr_create(int B, int H, int W, float thr, int border_rm, float temperature, int precision, int reserved_sms,
                     mfr_loftr** out) {
  if (!out) return MFR_ERR_ARG;
  mfr::LoftrEngine* e = nullptr;
  int rc = mfr::loftr_create(B, H, W, thr, border_rm, temperature, precision, reserved_sms, &e);
  if (rc != MFR_OK) return rc;
  *out = new mfr_loftr{e};
  return MFR_OK;
}
void mfr_loftr_destroy(mfr_loftr* h) {
  if (!h) return;
  mfr::loftr_destroy(h->e);
  delete h;
}
int mfr_loftr_num_weights(const mfr_loftr* h) { return core(h).weights.count(); }
const char* mfr_loftr_weight_name(const mfr_loftr* h, int i) { return core(h).weights.name(i); }
long long mfr_loftr_weight_numel(const mfr_loftr* h, int i) { return core(h).weights.numel(i); }
int mfr_loftr_set_weight(mfr_loftr* h, int i, const float* host, long long numel, void* stream) {
  return core(h).weights.set(i, host, numel, static_cast<cudaStream_t>(stream));
}
int mfr_loftr_forward(mfr_loftr* h, const float* img0, const float* img1, int src_h, int src_w, void* stream) {
  return mfr::loftr_forward(h->e, img0, img1, src_h, src_w, static_cast<cudaStream_t>(stream));
}
int mfr_loftr_set_map(mfr_loftr* h, const float* img0, int src_h, int src_w, void* stream) {
  if (!h || !img0) return MFR_ERR_ARG;
  return mfr::loftr_set_map(h->e, img0, src_h, src_w, static_cast<cudaStream_t>(stream));
}
int mfr_loftr_forward_shared(mfr_loftr* h, const float* img1, int src_h, int src_w, void* stream) {
  if (!h || !img1) return MFR_ERR_ARG;
  return mfr::loftr_forward_shared(h->e, img1, src_h, src_w, static_cast<cudaStream_t>(stream));
}
void mfr_loftr_set_graph(mfr_loftr* h, int enabled) { if (h) core(h).use_graph = enabled != 0; }
int mfr_loftr_get_outputs(mfr_loftr* h, mfr_loftr_outputs* out) {
  if (!h || !out) return MFR_ERR_ARG;
  mfr::loftr_outputs(h->e, out);
  return MFR_OK;
}
int mfr_loftr_debug_tensor(mfr_loftr* h, const char* name, float** ptr, long long* numel) {
  if (!h) return MFR_ERR_ARG;
  return core(h).mem.debug_tensor(name, ptr, numel);
}
int mfr_loftr_num_kernels(const mfr_loftr* h) { return core(h).steps.size(); }
int mfr_loftr_num_launches(const mfr_loftr* h) { return core(h).steps.launches(); }
int mfr_loftr_profile(mfr_loftr* h, const float* img0, const float* img1, int src_h, int src_w, void* stream,
                      int max_steps, float* ms, double* flops, int* kinds, char* names) {
  return mfr::loftr_profile(h->e, img0, img1, src_h, src_w, static_cast<cudaStream_t>(stream), max_steps, ms, flops,
                            kinds, names);
}
const char* mfr_loftr_step_name(const mfr_loftr* h, int i) {
  if (!h || i < 0 || i >= core(h).steps.size()) return nullptr;
  return core(h).steps.steps[i].name.c_str();
}
int mfr_loftr_run_steps(mfr_loftr* h, int begin, int end, void* stream) {
  if (!h) return MFR_ERR_ARG;
  return mfr::loftr_run_steps(h->e, begin, end, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------ SuperPoint + SuperGlue
struct mfr_spsg { mfr::SpsgEngine* e; };
int mfr_spsg_create_ex(int B, int H, int W, int max_keypoints, int nms_radius, float keypoint_threshold,
                       int remove_borders, int sinkhorn_iterations, float match_threshold, int precision,
                       mfr_spsg** out) {
  if (!out) return MFR_ERR_ARG;
  mfr::SpsgEngine* e = nullptr;
  int rc = mfr::spsg_create(B, H, W, max_keypoints, nms_radius, keypoint_threshold, remove_borders,
                            sinkhorn_iterations, match_threshold, precision, &e);
  if (rc != MFR_OK) return rc;
  *out = new mfr_spsg{e};
  return MFR_OK;
}
int mfr_spsg_create(int B, int H, int W, int max_keypoints, int nms_radius, float keypoint_threshold,
                    int remove_borders, int sinkhorn_iterations, float match_threshold, mfr_spsg** out) {
  return mfr_spsg_create_ex(B, H, W, max_keypoints, nms_radius, keypoint_threshold, remove_borders,
                            sinkhorn_iterations, match_threshold, MFR_PRECISION_TF32, out);
}
void mfr_spsg_destroy(mfr_spsg* h) { if (h) { mfr::spsg_destroy(h->e); delete h; } }
int mfr_spsg_num_weights(const mfr_spsg* h) { return core(h).weights.count(); }
const char* mfr_spsg_weight_name(const mfr_spsg* h, int i) { return core(h).weights.name(i); }
long long mfr_spsg_weight_numel(const mfr_spsg* h, int i) { return core(h).weights.numel(i); }
int mfr_spsg_set_weight(mfr_spsg* h, int i, const float* host, long long numel, void* stream) {
  return core(h).weights.set(i, host, numel, static_cast<cudaStream_t>(stream));
}
int mfr_spsg_forward(mfr_spsg* h, const float* img0, const float* img1, void* stream) {
  return mfr::spsg_forward(h->e, img0, img1, static_cast<cudaStream_t>(stream));
}
int mfr_spsg_set_map(mfr_spsg* h, const float* img0, void* stream) {
  if (!h || !img0) return MFR_ERR_ARG;
  return mfr::spsg_set_map(h->e, img0, static_cast<cudaStream_t>(stream));
}
int mfr_spsg_forward_shared(mfr_spsg* h, const float* img1, void* stream) {
  if (!h || !img1) return MFR_ERR_ARG;
  return mfr::spsg_forward_shared(h->e, img1, static_cast<cudaStream_t>(stream));
}
void mfr_spsg_set_graph(mfr_spsg* h, int enabled) { if (h) core(h).use_graph = enabled != 0; }
int mfr_spsg_get_outputs(mfr_spsg* h, mfr_spsg_outputs* out) {
  if (!h || !out) return MFR_ERR_ARG;
  mfr::spsg_outputs(h->e, out);
  return MFR_OK;
}
int mfr_spsg_debug_tensor(mfr_spsg* h, const char* name, float** ptr, long long* numel) {
  if (!h) return MFR_ERR_ARG;
  return core(h).mem.debug_tensor(name, ptr, numel);
}
int mfr_spsg_num_launches(const mfr_spsg* h) { return core(h).steps.launches(); }
int mfr_spsg_forward_superglue(mfr_spsg* h, const int* counts, const float* keypoints, const float* scores,
                               const float* descriptors, void* stream) {
  return mfr::spsg_forward_superglue(h->e, counts, keypoints, scores, descriptors, static_cast<cudaStream_t>(stream));
}

int mfr_coarse_match(const float* sim, int B, int h_c, int w_c, float thr, int border_rm, float scale,
                     int input_is_conf, int* count, int* offsets, int* b_ids, int* i_ids, int* j_ids,
                     float* mconf, float* mkpts0_c, float* mkpts1_c, void* stream) {
  if (!sim || B < 1 || h_c < 1 || w_c < 1) return MFR_ERR_ARG;
  const int L = h_c * w_c, splits = mfr::coarse_match_splits(B, L);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  mfr::CoarseMatchBuffers b;
  int rc = mfr::coarse_match_alloc(B, L, splits, &b);
  if (rc != MFR_OK) return rc;
  rc = mfr::coarse_match(sim, b, B, L, h_c, w_c, thr, border_rm, scale, splits, st, input_is_conf != 0);
  const size_t BL = static_cast<size_t>(B) * L;
  if (rc == MFR_OK) {
    cudaMemcpyAsync(count, b.m_total, 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(offsets, b.m_offsets, (B + 1) * 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(b_ids, b.b_ids, BL * 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(i_ids, b.i_ids, BL * 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(j_ids, b.j_ids, BL * 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(mconf, b.mconf, BL * 4, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(mkpts0_c, b.mkpts0_c, BL * 8, cudaMemcpyDeviceToDevice, st);
    cudaMemcpyAsync(mkpts1_c, b.mkpts1_c, BL * 8, cudaMemcpyDeviceToDevice, st);
  }
  cudaStreamSynchronize(st);
  mfr::coarse_match_free(&b);
  return rc;
}

int mfr_knn2_l2(const float* query, int nq, const float* train, int nt, int dim, int* idx1, float* dist1,
                int* idx2, float* dist2, void* stream) {
  return mfr::knn2_l2(query, nq, train, nt, dim, idx1, dist1, idx2, dist2, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------ SIFT
struct mfr_sift { mfr::SiftEngine* e; };
int mfr_sift_create(int B, int H, int W, int nfeatures, int max_candidates, int root_sift, mfr_sift** out) {
  if (!out) return MFR_ERR_ARG;
  mfr::SiftEngine* e = nullptr;
  int rc = mfr::sift_create(B, H, W, nfeatures, max_candidates, root_sift, &e);
  if (rc != MFR_OK) return rc;
  *out = new mfr_sift{e};
  return MFR_OK;
}
void mfr_sift_destroy(mfr_sift* h) { if (h) { mfr::sift_destroy(h->e); delete h; } }
int mfr_sift_detect(mfr_sift* h, const unsigned char* imgs, void* stream) {
  if (!h) return MFR_ERR_ARG;
  return mfr::sift_detect(h->e, imgs, static_cast<cudaStream_t>(stream));
}
void mfr_sift_set_graph(mfr_sift* h, int enabled) { if (h) core(h).use_graph = enabled != 0; }
int mfr_sift_get_outputs(mfr_sift* h, mfr_sift_outputs* out) {
  if (!h || !out) return MFR_ERR_ARG;
  mfr::sift_outputs(h->e, out);
  return MFR_OK;
}
int mfr_sift_match_pairs(mfr_sift* h, float ratio, float* kpts0, float* kpts1, int* offsets, void* stream) {
  if (!h) return MFR_ERR_ARG;
  return mfr::sift_match_pairs(h->e, ratio, kpts0, kpts1, offsets, static_cast<cudaStream_t>(stream));
}
int mfr_sift_debug_tensor(mfr_sift* h, const char* name, float** ptr, long long* numel) {
  if (!h) return MFR_ERR_ARG;
  return core(h).mem.debug_tensor(name, ptr, numel);
}
int mfr_sift_profile(mfr_sift* h, const unsigned char* imgs, float* ms, void* stream) {
  if (!h) return MFR_ERR_ARG;
  return mfr::sift_profile(h->e, imgs, ms, static_cast<cudaStream_t>(stream));
}

struct mfr_sift_pairs { mfr::SiftPairs* e; };
int mfr_sift_pairs_create(int P, int H, int W, int nfeatures, int max_candidates, int root_sift, float ratio,
                          mfr_sift_pairs** out) {
  if (!out) return MFR_ERR_ARG;
  mfr::SiftPairs* e = nullptr;
  int rc = mfr::sift_pairs_create(P, H, W, nfeatures, max_candidates, root_sift, ratio, &e);
  if (rc != MFR_OK) return rc;
  *out = new mfr_sift_pairs{e};
  return MFR_OK;
}
void mfr_sift_pairs_destroy(mfr_sift_pairs* h) { if (h) { mfr::sift_pairs_destroy(h->e); delete h; } }
void mfr_sift_pairs_set_graph(mfr_sift_pairs* h, int enabled) { if (h) core(h).use_graph = enabled != 0; }
int mfr_sift_forward_pairs(mfr_sift_pairs* h, const unsigned char* img0, const unsigned char* img1, void* stream) {
  if (!h) return MFR_ERR_ARG;
  return mfr::sift_forward_pairs(h->e, img0, img1, static_cast<cudaStream_t>(stream));
}
int mfr_sift_set_map(mfr_sift_pairs* h, const unsigned char* img0, void* stream) {
  if (!h) return MFR_ERR_ARG;
  return mfr::sift_pairs_set_map(h->e, img0, static_cast<cudaStream_t>(stream));
}
int mfr_sift_forward_shared(mfr_sift_pairs* h, const unsigned char* img1, void* stream) {
  if (!h) return MFR_ERR_ARG;
  return mfr::sift_forward_shared(h->e, img1, static_cast<cudaStream_t>(stream));
}
int mfr_sift_get_pair_outputs(mfr_sift_pairs* h, mfr_sift_pair_outputs* out) {
  if (!h || !out) return MFR_ERR_ARG;
  mfr::sift_pair_outputs(h->e, out);
  return MFR_OK;
}

// ------------------------------------------------------------------------------------------ pose back end
struct mfr_pose_solver { mfr::PoseSolver* s; };

int mfr_pose_solver_create(int max_pairs, int max_pts_per_pair, int max_hypotheses, mfr_pose_solver** out) {
  if (!out) return MFR_ERR_ARG;
  mfr::PoseSolver* s = nullptr;
  int rc = mfr::pose_solver_create(max_pairs, max_pts_per_pair, max_hypotheses, &s);
  if (rc != MFR_OK) return rc;
  *out = new mfr_pose_solver{s};
  return MFR_OK;
}
void mfr_pose_solver_destroy(mfr_pose_solver* s) {
  if (!s) return;
  mfr::pose_solver_destroy(s->s);
  delete s;
}
int mfr_pose_solver_debug_tensor(mfr_pose_solver* s, const char* name, void** ptr, long long* words) {
  if (!s) return MFR_ERR_ARG;
  return mfr::pose_solver_debug_tensor(s->s, name, ptr, words);
}
int mfr_emat_ransac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                    const float* K0, const float* K1, float pix_threshold, int num_hyp,
                    unsigned long long seed, int lo_enabled, float* R, float* t, int* n_inliers,
                    unsigned char* mask, void* stream) {
  return mfr::emat_ransac(s->s, kpts0, kpts1, offsets, P, K0, K1, pix_threshold, num_hyp, seed, lo_enabled, R,
                          t, n_inliers, mask, static_cast<cudaStream_t>(stream));
}
int mfr_scale_from_depth(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                         const float* K0, const float* K1, const unsigned char* mask, const double* Rd,
                         const double* td, const float* depth0, const float* depth1, int H, int W,
                         float scale_threshold, float* R_out, float* t_metric, int* inliers, void* stream) {
  return mfr::scale_from_depth(s->s, kpts0, kpts1, offsets, P, K0, K1, mask, Rd, td, depth0, depth1, H, W,
                               scale_threshold, R_out, t_metric, inliers, static_cast<cudaStream_t>(stream));
}
int mfr_pnp_ransac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                   const float* K0, const float* K1, const float* depth0, int H, int W, int num_hyp,
                   float reproj_threshold, unsigned long long seed, float* R, float* t, int* n_inliers,
                   unsigned char* mask, void* stream) {
  return mfr::pnp_ransac(s->s, kpts0, kpts1, offsets, P, K0, K1, depth0, H, W, num_hyp, reproj_threshold, seed,
                         R, t, n_inliers, mask, static_cast<cudaStream_t>(stream));
}
int mfr_emat_ransac_escalate(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                             const float* K0, const float* K1, float pix_threshold, int num_hyp,
                             unsigned long long seed, int lo_enabled, float* R, float* t, int* n_inliers,
                             unsigned char* mask, double confidence, int max_hyp, int* budgets_out, void* stream) {
  if (!s) return MFR_ERR_ARG;
  return mfr::emat_ransac_escalate(s->s, kpts0, kpts1, offsets, P, K0, K1, pix_threshold, num_hyp, seed, lo_enabled, R,
                                   t, n_inliers, mask, confidence, max_hyp, budgets_out, static_cast<cudaStream_t>(stream));
}
int mfr_emat_magsac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                    const float* K0, const float* K1, float pix_threshold, int num_hyp, unsigned long long seed, float* R,
                    float* t, int* n_inliers, unsigned char* mask, double confidence, int max_hyp, int* budgets_out,
                    void* stream) {
  if (!s) return MFR_ERR_ARG;
  return mfr::emat_magsac(s->s, kpts0, kpts1, offsets, P, K0, K1, pix_threshold, num_hyp, seed, R, t, n_inliers, mask,
                          confidence, max_hyp, budgets_out, static_cast<cudaStream_t>(stream));
}
int mfr_pnp_ransac_escalate(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                            const float* K0, const float* K1, const float* depth0, int H, int W, int num_hyp,
                            float reproj_threshold, unsigned long long seed, float* R, float* t, int* n_inliers,
                            unsigned char* mask, double confidence, int max_hyp, int* budgets_out, void* stream) {
  if (!s) return MFR_ERR_ARG;
  return mfr::pnp_ransac_escalate(s->s, kpts0, kpts1, offsets, P, K0, K1, depth0, H, W, num_hyp, reproj_threshold, seed,
                                  R, t, n_inliers, mask, confidence, max_hyp, budgets_out, static_cast<cudaStream_t>(stream));
}

int mfr_procrustes_ransac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                          const float* K0, const float* K1, const float* depth0, const float* depth1, int H, int W,
                          int num_hyp, float max_corr_dist, unsigned long long seed, float* R, float* t,
                          int* n_inliers, void* stream) {
  return mfr::procrustes_ransac(s->s, kpts0, kpts1, offsets, P, K0, K1, depth0, depth1, H, W, num_hyp, max_corr_dist,
                                seed, R, t, n_inliers, static_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------ host test hooks
int mfr_host_five_point(const double* x0, const double* x1, double* E_out) {
  return mfr::geo::five_point(reinterpret_cast<const double(*)[2]>(x0), reinterpret_cast<const double(*)[2]>(x1),
                              reinterpret_cast<double(*)[9]>(E_out));
}
int mfr_host_p3p(const double* X, const double* f, double* R_out, double* t_out) {
  return mfr::geo::p3p(reinterpret_cast<const double(*)[3]>(X), reinterpret_cast<const double(*)[3]>(f),
                       reinterpret_cast<double(*)[9]>(R_out), reinterpret_cast<double(*)[3]>(t_out));
}
int mfr_host_kabsch(double n, const double* sum_p, const double* sum_q, const double* sum_pq, double* R, double* t) {
  return mfr::geo::kabsch_from_sums(n, sum_p, sum_q, sum_pq, R, t) ? 1 : 0;
}
int mfr_host_poly_real_roots(const double* coef, int deg, double* roots) {
  if (deg < 1 || deg > mfr::geo::kMaxDeg) return -1;
  return mfr::geo::poly_real_roots(coef, deg, roots);
}
int mfr_host_decompose_essential(const double* E, double* R1, double* R2, double* t) {
  mfr::geo::decompose_essential(E, R1, R2, t);
  return MFR_OK;
}
int mfr_host_ransac_satisfied(double confidence, int n_inliers, int n_points, int budget, int max_budget, int sample_size) {
  return mfr::geo::ransac_satisfied(confidence, n_inliers, n_points, budget, max_budget, sample_size) ? 1 : 0;
}
int mfr_host_magsac_loss(double r, double sigma_max, double* rho, double* w) {
  if (!(sigma_max > 0.0) || !rho || !w) return MFR_ERR_ARG;
  mfr::geo::magsac_loss_sq(r * r, sigma_max, rho, w);
  return MFR_OK;
}
int mfr_host_jpeg_decode(const unsigned char* data, long long length, int rgb, unsigned char* dst, int width, int height) {
  if (!data || length <= 0 || !dst) return MFR_ERR_ARG;
  return mfr::jpeg_host_decode(data, static_cast<size_t>(length), rgb, dst, width, height);
}
// lib/datasets/utils.py:77-81 (read_depth_image), serially on the CPU
int mfr_host_png_decode(const unsigned char* data, long long length, int out_kind, void* dst, int width, int height) {
  if (!data || length <= 0 || !dst) return MFR_ERR_ARG;
  return mfr::png_host_decode(data, static_cast<size_t>(length), out_kind, dst, width, height);
}

// ------------------------------------------------------------------------------------------ debug probes
int mfr_debug_png_kernel_ms(mfr_png_decoder* dec, float* ms) {
  if (!dec || !ms) return MFR_ERR_ARG;
  return mfr::png_decoder_kernel_ms(dec->d, ms);
}
float mfr_debug_time_conv(const float* x, int N, int H, int W, int Cin, const float* w, int Cout, int R,
                          int stride, float* out, int iters, int flags, const float* residual) {
  mfr::ConvGemmDesc d{};
  d.x = x; d.N = N; d.H = H; d.W = W; d.Cin = Cin; d.ldx = Cin;
  d.w = w; d.Cout = Cout; d.R = R; d.S = R; d.stride = stride; d.pad = R / 2;
  d.act = 1; d.alpha = 1.f; d.out = out; d.ldo = Cout; d.ldr = Cout;
  d.in_bf16 = flags & 1; d.out_bf16 = (flags >> 1) & 1; d.residual = residual;
  if (flags & 4) {   // channel strides padded to multiples of 8 elements (how the engine stores the 196-channel maps)
    d.ldx = (Cin + 7) / 8 * 8; d.ldw = d.ldx; d.ldo = (Cout + 7) / 8 * 8; d.ldr = d.ldo;
  }
  mfr::ConvGemmParams p;
  if (mfr::conv_gemm_build(d, &p) != MFR_OK) return -1.f;
  return mfr::conv_gemm_time_prebuilt(p, iters, nullptr);
}

int mfr_stem_conv7x7(const float* img, const float* w, const float* bias, void* out, int NI, int H, int W, int out_bf16,
                     int exact_fp32, void* stream) {
  if (!img || !w || !bias || !out || NI <= 0 || H < 7 || W < 7) return MFR_ERR_ARG;
  return mfr::stem_conv7x7(img, w, bias, static_cast<float*>(out), NI, H, W, static_cast<cudaStream_t>(stream), out_bf16, exact_fp32);
}

int mfr_linear_attention(const void* q, const void* k, const void* v, void* msg, int n, int L, int S, int windows,
                         int bf16, void* stream) {
  if (!q || !k || !v || !msg || n <= 0) return MFR_ERR_ARG;
  if (bf16 != 0 && bf16 != 2) return MFR_ERR_UNSUPPORTED;   // bf16 takes raw q, k: pre-mapped ones would be mapped twice
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (windows) {
    int* cnt = nullptr;
    if (cudaMalloc(&cnt, sizeof(int)) != cudaSuccess) return MFR_ERR_CUDA;
    cudaMemcpyAsync(cnt, &n, sizeof(int), cudaMemcpyHostToDevice, st);
    const int r = mfr::linear_attention_windows(q, 128, k, 128, v, 128, msg, 128, cnt, n, 25, st, bf16);
    cudaStreamSynchronize(st);
    cudaFree(cnt);
    return r;
  }
  if (L <= 0 || S <= 0) return MFR_ERR_ARG;
  const int splits = std::max(1, std::min((S + 63) / 64, (2 * mfr::sm_count() + n - 1) / n));
  float *kv_part = nullptr, *kv = nullptr;
  if (cudaMalloc(&kv_part, static_cast<size_t>(n) * splits * 8448 * sizeof(float)) != cudaSuccess) return MFR_ERR_CUDA;
  if (cudaMalloc(&kv, static_cast<size_t>(n) * 8448 * sizeof(float)) != cudaSuccess) { cudaFree(kv_part); return MFR_ERR_CUDA; }
  const int r = mfr::linear_attention_long(q, 256, k, 256, v, 256, msg, 256, kv_part, kv, n, L, S, 8, 32, splits, st, bf16);
  cudaStreamSynchronize(st);
  cudaFree(kv_part); cudaFree(kv);
  return r;
}

int mfr_superglue_attention(const void* qkv, long long ldq, const int* counts, int n_img, int max_kp, int cross,
                            void* msg, long long ldo, void* stream) {
  mfr::SgAttentionParams p;
  const int r = mfr::sg_attention_build(qkv, ldq, counts, n_img, max_kp, cross, msg, ldo, &p);
  if (r != MFR_OK) return r;
  return mfr::sg_attention_launch(p, static_cast<cudaStream_t>(stream));
}

int mfr_icp_refine(mfr_pose_solver* s, const float* depth0, const float* depth1, int H, int W, int P, const float* K0,
                   const float* K1, const float* R_in, const float* t_in, float max_corr_dist, int max_iterations,
                   float relative_fitness, float relative_rmse, float* R, float* t, int* n_inliers, void* stream) {
  if (!s || !depth0 || !depth1 || !K0 || !K1 || !R_in || !t_in || !R || !t || !n_inliers) return MFR_ERR_ARG;
  return mfr::icp_refine(s->s, depth0, depth1, H, W, P, K0, K1, R_in, t_in, max_corr_dist, max_iterations, relative_fitness,
                         relative_rmse, R, t, n_inliers, static_cast<cudaStream_t>(stream));
}

int mfr_resize_linear(const void* src, int src_is_u8, int src_w, int src_h, long long src_row_stride, int channels, float* dst,
                      int dst_w, int dst_h, int mode, float out_scale, int chw, void* stream) {
  return mfr::resize_linear(src, src_is_u8, src_w, src_h, src_row_stride, channels, dst, dst_w, dst_h, mode, out_scale, chw,
                            static_cast<cudaStream_t>(stream));
}
int mfr_jpeg_info(const unsigned char* data, long long length, int* width, int* height, int* components) {
  if (!data || length <= 0 || !width || !height || !components) return MFR_ERR_ARG;
  return mfr::jpeg_info(data, static_cast<size_t>(length), width, height, components);
}
int mfr_jpeg_decode(const unsigned char* data, long long length, int rgb, unsigned char* dst, int width, int height, void* stream) {
  if (!data || length <= 0 || !dst) return MFR_ERR_ARG;
  return mfr::jpeg_decode(data, static_cast<size_t>(length), rgb, dst, width, height, static_cast<cudaStream_t>(stream));
}
int mfr_jpeg_decoder_create(int max_images, long long max_bytes, long long max_pixels, mfr_jpeg_decoder** out) {
  if (!out) return MFR_ERR_ARG;
  *out = nullptr;
  mfr::JpegDecoder* d = nullptr;
  const int rc = mfr::jpeg_decoder_create(max_images, max_bytes, max_pixels, &d);
  if (rc != MFR_OK) return rc;
  *out = new mfr_jpeg_decoder{d};
  return MFR_OK;
}
void mfr_jpeg_decoder_destroy(mfr_jpeg_decoder* dec) {
  if (!dec) return;
  mfr::jpeg_decoder_destroy(dec->d);
  delete dec;
}
int mfr_jpeg_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* status) {
  if (n < 0 || (n > 0 && (!data || !lengths || !width || !height || !status))) return MFR_ERR_ARG;
  mfr::jpeg_batch_info(data, lengths, n, width, height, status);
  return MFR_OK;
}
int mfr_jpeg_decode_batch(mfr_jpeg_decoder* dec, const unsigned char* const* data, const long long* lengths, int n, int rgb,
                          unsigned char* const* dst, int* status, void* stream) {
  if (!dec) return MFR_ERR_ARG;
  return mfr::jpeg_decode_batch(dec->d, data, lengths, n, rgb, dst, status, static_cast<cudaStream_t>(stream));
}
// lib/datasets/utils.py:77-81: read_depth_image's cv2.imread(path, IMREAD_UNCHANGED) of a 16-bit depth PNG
int mfr_png_info(const unsigned char* data, long long length, int* width, int* height, int* bit_depth) {
  if (!data || length <= 0 || !width || !height || !bit_depth) return MFR_ERR_ARG;
  return mfr::png_info(data, static_cast<size_t>(length), width, height, bit_depth);
}
// lib/datasets/utils.py:77-81
int mfr_png_decoder_create(int max_images, long long max_bytes, long long max_pixels, mfr_png_decoder** out) {
  if (!out) return MFR_ERR_ARG;
  *out = nullptr;
  mfr::PngDecoder* d = nullptr;
  const int rc = mfr::png_decoder_create(max_images, max_bytes, max_pixels, &d);
  if (rc != MFR_OK) return rc;
  *out = new mfr_png_decoder{d};
  return MFR_OK;
}
void mfr_png_decoder_destroy(mfr_png_decoder* dec) {
  if (!dec) return;
  mfr::png_decoder_destroy(dec->d);
  delete dec;
}
// lib/datasets/utils.py:77-81
int mfr_png_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* bit_depth,
                       int* status) {
  if (n < 0 || (n > 0 && (!data || !lengths || !width || !height || !bit_depth || !status))) return MFR_ERR_ARG;
  mfr::png_batch_info(data, lengths, n, width, height, bit_depth, status);
  return MFR_OK;
}
// lib/datasets/utils.py:77-81: out_kind 0 = cv2.imread(IMREAD_UNCHANGED), 1 = that / 1000 as float32
int mfr_png_decode_batch(mfr_png_decoder* dec, const unsigned char* const* data, const long long* lengths, int n, int out_kind,
                         void* const* dst, int* status, void* stream) {
  if (!dec) return MFR_ERR_ARG;
  return mfr::png_decode_batch(dec->d, data, lengths, n, out_kind, dst, status, static_cast<cudaStream_t>(stream));
}

int mfr_pose_metrics(const double* q_gt, const double* t_gt, const double* q_est, const double* t_est, const double* K, int W,
                     int H, int n, double* trans_err, double* rot_err, double* reproj_err, void* stream) {
  if (n < 0 || (n > 0 && (!q_gt || !t_gt || !q_est || !t_est || !K || !trans_err || !rot_err || !reproj_err))) return MFR_ERR_ARG;
  return mfr::pose_metrics(q_gt, t_gt, q_est, t_est, K, W, H, n, trans_err, rot_err, reproj_err, static_cast<cudaStream_t>(stream));
}

int mfr_encoder_tail(const void* msg, void* xb, float* x, const void* w_merge, const void* w_mlp0, const void* w_mlp2,
                     const float* g1, const float* b1, const float* g2, const float* b2, int C, int n_blocks,
                     long long rows_cap, const int* dyn_rows, int iters, void* stream) {
  if (!msg || !xb || !x || !w_merge || !w_mlp0 || !w_mlp2 || !g1 || !b1 || !g2 || !b2 || iters < 1) return MFR_ERR_ARG;
  mfr::EncoderTailDesc d{};
  d.msg = msg; d.ld_msg = C; d.xb_in = xb; d.ld_xb = 2 * C; d.w_merge = w_merge; d.w_mlp0 = w_mlp0; d.w_mlp2 = w_mlp2;
  d.g1 = g1; d.b1 = b1; d.g2 = g2; d.b2 = b2; d.x = x; d.ldx = 2 * C; d.C = C; d.n_img = n_blocks; d.rows_cap = rows_cap;
  d.dyn_rows = dyn_rows;
  mfr::EncoderTailParams p;
  int rc = mfr::encoder_tail_build(d, &p);
  for (int i = 0; i < iters && rc == MFR_OK; ++i) rc = mfr::encoder_tail_launch(p, static_cast<cudaStream_t>(stream));
  return rc;
}

}  // extern "C"
