// SIMT kernels of the LoFTR matcher that are not GEMM-shaped (launch wrappers).
// All tensors are fp32, channel-last; `ld*` are row strides in floats.
#pragma once
#include "common.cuh"

namespace mfr {

// stem: conv7x7 stride 2 pad 3, 1 -> 128 channels, folded BN bias, ReLU (resnet_fpn.py:60-62,102)
// exact_fp32: plain fp32 FMA kernel instead of the tensor-core one (bf16 hi/lo split, ~2^-16 relative)
int stem_conv7x7(const float* img, const float* w /*[128][49]*/, const float* bias, float* out,
                 int NI, int H, int W, cudaStream_t st, int out_bf16 = 0, int exact_fp32 = 0);

// dst[n,y,x,:] += bilinear_x2_align_corners(src)[n,y,x,:]   (resnet_fpn.py:110,114)
// pixel strides lds / ldd in elements; src / dst fp32 or bf16
int upsample2x_add(const void* src, void* dst, int N, int Hs, int Ws, int C, int lds, int ldd, int src_bf16,
                   int dst_bf16, cudaStream_t st);
// fp32 [rows][cin] -> bf16 [rows][cin_pad], zero padded
int weights_to_bf16(const float* src, void* dst, size_t rows, int cin, int cin_pad, cudaStream_t st);

// tok[n,l,0:C] = feat[n,l,:] + pe[l,:]   (loftr.py:58-59, position_encoding.py:42)
int posenc_tokens(const float* feat, const float* pe, float* tok, long long ldt, int N, int L, int C,
                  cudaStream_t st);

// Linear attention (linear_attention.py:31-45) for a few long sequences (coarse level).
//   K,V: [n][S][H*D] (row strides ldk, ldv), already elu+1'd K.  Q: [n][L][H*D].
//   msg[n,l,h,:] = (Q . KV) / (Q . Ksum + eps),  KV = sum_s K^T (V/S) * S
// scratch: kv_part [n][H][splits][(D+1)*D], kv [n][H][(D+1)*D]
// bf16 != 0: Q / K / V / msg are bf16 (strides in elements), sums stay fp32, and Q and K are the raw projections:
// the kernels apply elu(x) + 1 themselves
int linear_attention_long(const void* Q, long long ldq, const void* K, long long ldk, const void* V,
                          long long ldv, void* msg, long long ldm, float* kv_part, float* kv, int n,
                          int L, int S, int heads, int dim, int splits, cudaStream_t st, int bf16 = 0);

// Linear attention for many short sequences (fine level): items of `T` tokens (T <= 32), C = 128,
// 8 heads x 16. x-side item i attends to src-side item i. n_items read from device (*n_items_dev).
// bf16 as for linear_attention_long.
int linear_attention_windows(const void* Q, long long ldq, const void* K, long long ldk, const void* V,
                             long long ldv, void* msg, long long ldm, const int* n_items_dev,
                             int max_items, int T, cudaStream_t st, int bf16 = 0);

// out[r,:] = (res ? res[r,:] : 0) + LayerNorm(in[r,:]) * gamma + beta, C in {128, 256}; rows may be
// limited by *dyn_rows (device) when non-null.
int layernorm_rows(const float* in, long long ldi, const float* gamma, const float* beta,
                   const float* res, long long ldr, float* out, long long ldo, long long rows, int C,
                   const int* dyn_rows, cudaStream_t st);
// dst16[row][0..C) = bf16(src[row][0..C)); rows optionally capped by *dyn_rows
int rows_to_bf16(const float* src, long long lds, void* dst, long long ldd, long long rows, int C, const int* dyn_rows,
                 cudaStream_t st);

// dst[k * bytes .. (k + 1) * bytes) = src[0 .. bytes) for k < copies (16-byte aligned, bytes a multiple of 16)
int broadcast_copies(const void* src, long long bytes, void* dst, int copies, cudaStream_t st);

// 3xTF32 operand split: dst[img][row][0:3C] = [hi | lo | hi] (pattern 0) or [hi | hi | lo] (pattern 1) of
// src[img][row][0:C]; hi = tf32(x), lo = tf32(x - hi). Rows per image optionally capped by *dyn_rows.
int rows_split3(const float* src, long long lds, long long src_img_stride, float* dst, long long rows_per_img,
                int images, int C, int pattern, const int* dyn_rows, cudaStream_t st);

// ---- coarse matching on the materialised similarity matrix S [B][L][L] (coarse_matching.py) ----
struct CoarseMatchBuffers {
  float* row_max; float* row_rsum;     // [B][L]  row softmax stats (max, 1/sum)
  float* col_max; float* col_rsum;     // [B][L]
  float* col_part;                     // [B][splits][L][2] scratch
  float* rconf_max; int* rconf_arg; int* rconf_ties;   // [B][L] row max of conf, first argmax, #ties
  float* cconf_max;                    // [B][L] column max of conf
  int* jsel;                           // [B][L] selected column or -1
  // compacted outputs (batch-global, ordered by (b, i))
  int* m_total;                        // [4]: {Mtot, 2*Mtot, 25*Mtot, 50*Mtot}
  int* m_offsets;                      // [B+1]
  int* b_ids; int* i_ids; int* j_ids;  // [B*L]
  float* mconf;                        // [B*L]
  float* mkpts0_c; float* mkpts1_c;    // [B*L][2]
};
int coarse_match(const float* S, CoarseMatchBuffers bufs, int B, int L, int h_c, int w_c, float thr,
                 int border, float scale, int splits, cudaStream_t st, bool input_is_conf = false);
// scratch + output buffers for a standalone call (freed with coarse_match_free)
// row slabs per pair such that all pairs together give ~2 blocks per SM
int coarse_match_splits(int B, int L);
int coarse_match_alloc(int B, int L, int splits, CoarseMatchBuffers* out);
void coarse_match_free(CoarseMatchBuffers* b);

// ---- fine level ----
// cin[(s*Mcap + m), 0:256] = feat_c{s}[b, i or j, :]   (fine_preprocess.py:51-52), tokens ld = ldt
int fine_gather_coarse(const float* tok, long long ldt, int B, int L, const int* b_ids, const int* i_ids,
                       const int* j_ids, const int* m_total, int Mcap, float* cin, cudaStream_t st);
// win[(s*Mcap + m)*25 + tap, 0:128] = 5x5 stride-4 window of feat_f (zero padded), [128:256] = cproj.
// Side s reads the fine map of pair b at featf_s + b * img_stride_s ([Hf][Wf][128] fp32); a stride of 0 makes every
// pair read the same map.
int fine_gather_windows(const float* featf0, long long img_stride0, const float* featf1, long long img_stride1, int Hf,
                        int Wf, int w_c, const int* b_ids, const int* i_ids, const int* j_ids, const int* m_total,
                        int Mcap, const float* cproj, float* win, cudaStream_t st);
// fine_matching.py:43-69: expectation over the 5x5 heat map, mkpts1_f = mkpts1_c + coords * 2 * scale
int fine_match(const float* f0, const float* f1, long long ldf, const float* mkpts1_c,
               const int* m_total, int Mcap, float scale_f, float* mkpts1_f, float* expec,
               cudaStream_t st);

}  // namespace mfr
