/* mfr_b200 — C ABI of the H100-native feature-matching + scale-from-depth hot path.
 *
 * Drop-in boundary for nianticlabs/map-free-reloc (reference paths are relative to that repo):
 * the reference has no FFI of its own (pure Python over torch / OpenCV wheels), so each entry
 * point below names the reference call it replaces. All pointers are DEVICE pointers unless
 * a parameter is documented as host memory; `stream` is a cudaStream_t passed as void*.
 * Every function returns MFR_OK (0) or an MFR_ERR_* code; geometric failures are reported the
 * way the reference does it: NaN-filled R/t and an inlier count of 0
 * (lib/models/matching/pose_solver.py:30-33).
 */
#ifndef MFR_B200_H_
#define MFR_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define MFR_OK 0
#define MFR_ERR_CUDA 1
#define MFR_ERR_ARG 2
#define MFR_ERR_UNSUPPORTED 3

/* activation codes for the fused conv/GEMM epilogue */
#define MFR_ACT_NONE 0
#define MFR_ACT_RELU 1
#define MFR_ACT_LEAKY 2 /* slope 0.01: nn.LeakyReLU() default, resnet_fpn.py:74,81 */
#define MFR_ACT_ELU1 3  /* elu(x)+1: linear_attention.py:10-11 */

/* Library / device probe. Returns the number of SMs of the current device (0 if no device). */
int mfr_version(void);
int mfr_device_sm_count(void);

/* Implicit-GEMM convolution on the Hopper tensor cores (wgmma, TF32 inputs, fp32 accumulate), NHWC.
 * Replaces torch's cuDNN conv2d / cuBLAS linear / einsum calls of the matcher networks:
 *   etc/feature_matching_baselines/LoFTR/src/loftr/backbone/resnet_fpn.py:5-12 (conv1x1/conv3x3),
 *   .../loftr_module/transformer.py:22-32 (Linear), .../utils/coarse_matching.py:113 (einsum).
 *   x   [N][H][W][Cin]  pixel stride ldx floats        w [Cout][R*S][Cin]
 *   out [N][Ho][Wo][Cout] pixel stride ldo floats; residual like out with stride ldr (or NULL)
 *   b_batched != 0: w is [N][Cout][Cin] and image n uses w[n] (batched X * Y^T).
 * out = act(alpha * conv(x, w) + bias + residual). R,S in {1,3}; stride in {1,2}. */
int mfr_conv2d_nhwc_tf32(const float* x, int N, int H, int W, int Cin, long long ldx,
                         const float* w, int Cout, int R, int S, int stride, int pad,
                         int b_batched, const float* bias, const float* residual, long long ldr,
                         int act, float alpha, float* out, long long ldo, void* stream);

/* Same op with bf16 operands (x, w as bf16 bits; bf16 wgmma, fp32 accumulate). ldx / ldw are
 * element strides with ldx*2 and ldw*2 multiples of 16 bytes (ldw = per-tap row stride of w, >= Cin).
 * out / residual are bf16 when out_bf16 != 0 (then Cout % 4 == 0), else fp32. bias is fp32.
 * Elements past Cout of an output row are not written. */
int mfr_conv2d_nhwc_bf16(const void* x, int N, int H, int W, int Cin, long long ldx, const void* w,
                         long long ldw, int Cout, int R, int S, int stride, int pad, const float* bias,
                         const void* residual, long long ldr, int act, float alpha, void* out,
                         long long ldo, int out_bf16, void* stream);

/* Stage entry for tests: a token GEMM (Linear layer) with a device row count, the form of the LoFTR fine-level
 * projections. n_img blocks of rows_cap token rows; block i computes rows r < *dyn_rows (read on the device at launch):
 *   out[i][r][co] = act(sum_ci x[i][r][ci] * w[co][ci] + bias[co]), co < Cout
 *   x   [n_img][rows_cap] rows of stride ldx elements, w [Cout] rows of stride ldw elements (0 = Cin); both bf16
 *       (bf16 wgmma) when in_bf16 != 0, else fp32 (TF32 wgmma); fp32 accumulate; bias fp32 or NULL
 *   out [n_img][rows_cap] rows of stride ldo elements, bf16 when out_bf16 != 0 (then Cout % 4 == 0), else fp32.
 * Rows at or past *dyn_rows and elements past Cout of a row are not written. */
int mfr_token_gemm_dyn_rows(const void* x, int n_img, int rows_cap, int Cin, long long ldx, const void* w,
                            long long ldw, int in_bf16, int Cout, const float* bias, int act, void* out,
                            long long ldo, int out_bf16, const int* dyn_rows, void* stream);

/* ---------------------------------------------------------------------------------------------
 * LoFTR matcher engine. Replaces LoFTR.forward of the reference
 * (etc/feature_matching_baselines/LoFTR/src/loftr/loftr.py:29-75) as driven by
 * LoFTR_matcher.match (etc/feature_matching_baselines/matchers.py:24-59), for B image pairs per
 * call. Images are device fp32 [B][src_h][src_w] in [0,1]; the engine frame [H][W] (multiples of 8)
 * is zero-padded on the right/bottom like the reference's ConstantPad2d (matchers.py:41-46). Weights are set tensor by tensor in the engine's own layout (BN folded,
 * conv weights [Cout][R*S][Cin]); mfr_loftr_weight_name/numel enumerate what is expected.
 * Outputs stay on the device (pointers owned by the engine), ordered by (pair, i) exactly like
 * torch.where in coarse_matching.py:194. */
typedef struct mfr_loftr mfr_loftr;
typedef struct {
  const int* m_total;    /* device int[4]: {M, 2M, 25M, 50M}, M = matches in the batch */
  const int* m_offsets;  /* device int[B+1] */
  const int* b_ids; const int* i_ids; const int* j_ids; /* device int[capacity] */
  const float* mconf;                                   /* device float[capacity] */
  const float* mkpts0_f; const float* mkpts1_f;         /* device float[capacity][2], pixels (x,y) */
  const float* mkpts1_c; const float* expec_f;          /* device float[capacity][2] / [capacity][3] */
  int capacity;
} mfr_loftr_outputs;

/* precision:
 *  0 TF32   fp32 storage everywhere, TF32 tensor-core inputs in every conv / linear / correlation GEMM (what
 *           torch + cuDNN do by default for the reference's convs on a GPU); attention, LayerNorm, softmax fp32.
 *  1 BF16   throughput mode. bf16 storage + kind::f16 MMAs (fp32 accumulate) for the ResNet-FPN maps, the token
 *           GEMM operands (q|k|v, mlp0 read a bf16 shadow of the token stream; q|k|v, attention message and MLP
 *           hidden tensors are stored in bf16), the linear attention and the coarse correlation operands. The two
 *           backbone outputs, the token residual stream, LayerNorm arithmetic, the similarity matrix S, dual
 *           softmax and fine matching stay fp32.
 *  2 FP32X3 fp32-faithful parity mode. fp32 storage; every GEMM (convs, linears, correlation) runs as a 3xTF32
 *           split product  A.B ~= Ahi.Bhi + Alo.Bhi + Ahi.Blo  (one tensor-core GEMM over 3x the K extent,
 *           ~2^-21 relative per product instead of TF32's 2^-11); stem, attention, LayerNorm in plain fp32. This
 *           is the mode whose match indices are compared with the reference's fp32 arithmetic. */
#define MFR_PRECISION_TF32 0
#define MFR_PRECISION_BF16 1
#define MFR_PRECISION_FP32X3 2
/* reserved_sms: the first four conv launches of every forward use at most (SM count - reserved_sms) SMs, so that
 * other work on the device, such as the pose solver of the previous batch on another stream, is not held up behind
 * them. 0 uses every SM; 0 <= reserved_sms < SM count, else MFR_ERR_ARG. The results do not depend on it. */
int mfr_loftr_create(int B, int H, int W, float thr, int border_rm, float temperature, int precision, int reserved_sms,
                     mfr_loftr** out);
void mfr_loftr_destroy(mfr_loftr* h);
int mfr_loftr_num_weights(const mfr_loftr* h);
const char* mfr_loftr_weight_name(const mfr_loftr* h, int i);
long long mfr_loftr_weight_numel(const mfr_loftr* h, int i);
int mfr_loftr_set_weight(mfr_loftr* h, int i, const float* host, long long numel, void* stream);
int mfr_loftr_forward(mfr_loftr* h, const float* img0, const float* img1, int src_h, int src_w,
                      void* stream);
/* Shared map frame (Map-free: every query of a scene is matched against the same reference image).
 * mfr_loftr_set_map encodes one map image img0 [src_h][src_w] (device float32) — backbone, position encoding and the
 * first coarse layer, which depend on that image alone — into buffers of its own; they stay valid until the next
 * set_map or weight upload, and a paired mfr_loftr_forward in between does not disturb them. Runs eagerly.
 * mfr_loftr_forward_shared(h, img1 [B][src_h][src_w]) then writes outputs bit-identical, in every precision, to
 * mfr_loftr_forward(h, img0 repeated B times, img1), and runs as its own CUDA graph. It returns MFR_ERR_ARG before any
 * set_map or when (src_h, src_w) differs from the map's. */
int mfr_loftr_set_map(mfr_loftr* h, const float* img0, int src_h, int src_w, void* stream);
int mfr_loftr_forward_shared(mfr_loftr* h, const float* img1, int src_h, int src_w, void* stream);
void mfr_loftr_set_graph(mfr_loftr* h, int enabled);
int mfr_loftr_get_outputs(mfr_loftr* h, mfr_loftr_outputs* out);
/* named intermediate buffers for stage-wise parity tests ("feat_c_backbone", "feat_f", "tok", "sim", ...). In every
 * engine's *_debug_tensor, numel counts 4-byte words, whatever the buffer's element type. */
int mfr_loftr_debug_tensor(mfr_loftr* h, const char* name, float** ptr, long long* numel);
int mfr_loftr_num_kernels(const mfr_loftr* h);  /* steps of the launch list per forward */
int mfr_loftr_num_launches(const mfr_loftr* h); /* kernel launches per forward */
/* Eager run with a CUDA-event pair around every step of the launch list (host arrays out):
 * ms[i] device time, flops[i] algorithmic FLOPs, kinds[i] 1 = tensor-core conv/GEMM, names 32 bytes each.
 * Returns the number of steps (or a negative MFR_ERR_*). */
int mfr_loftr_profile(mfr_loftr* h, const float* img0, const float* img1, int src_h, int src_w,
                      void* stream, int max_steps, float* ms, double* flops, int* kinds, char* names);
/* Stage-wise tests of buffers the forward overwrites later. mfr_loftr_step_name(h, i) is the name of step i of the
 * paired forward list ("stem", a conv's weight name such as "layer2.0.down", "upsample", "split3", ...), NULL when i is
 * out of range; the string lives as long as the engine. mfr_loftr_run_steps runs steps [begin, end) of that list
 * eagerly on the engine's buffers as the previous calls left them (the staged images of the last forward), after
 * rebuilding the derived weight copies as a forward does. MFR_ERR_ARG when the range is not within the list or a
 * weight has not been uploaded. Neither is used by the forward or its CUDA graph. */
const char* mfr_loftr_step_name(const mfr_loftr* h, int i);
int mfr_loftr_run_steps(mfr_loftr* h, int begin, int end, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SuperPoint + SuperGlue matcher engine. Replaces Matching.forward of the reference
 * (etc/feature_matching_baselines/SuperGlue/models/matching.py:56-84 = superpoint.py:145-202 x2 +
 * superglue.py:228-283) as driven by SuperGlue_matcher.match (matchers.py:93-120), B pairs per
 * call, images device fp32 [B][H][W] in [0,1]. Settings of matchers.py:65-71 are the defaults of
 * the Python wrapper (nms 4, threshold 0.005, border 4, 1024 keypoints, 20 Sinkhorn iterations,
 * match threshold 0.2). Weights in the engine's layout (mfr_spsg_weight_name enumerates them). */
typedef struct mfr_spsg mfr_spsg;
typedef struct {
  const int* counts;             /* device int[2B], pair-interleaved (2p = image0 of pair p) */
  const float* keypoints;        /* device float[2B][K][2] pixel (x,y) */
  const float* scores;           /* device float[2B][K] */
  const float* descriptors;      /* device float[2B][K][desc_ld] */
  int desc_ld;
  const int* matches0;           /* device int[B][K], -1 = unmatched (superglue.py:274) */
  const float* matching_scores0; /* device float[B][K] */
  const int* m_offsets;          /* device int[B+1] */
  const float* mkpts0; const float* mkpts1; /* device float[total][2], ordered by (pair, i) */
  int max_keypoints;
} mfr_spsg_outputs;
int mfr_spsg_create(int B, int H, int W, int max_keypoints, int nms_radius, float keypoint_threshold,
                    int remove_borders, int sinkhorn_iterations, float match_threshold, mfr_spsg** out);
/* same with the GEMM precision: MFR_PRECISION_TF32 (what mfr_spsg_create uses), MFR_PRECISION_FP32X3 (every conv /
 * linear / attention / score GEMM as a 3xTF32 split product: the fp32-faithful parity mode) or MFR_PRECISION_BF16
 * (throughput mode). In bf16 mode:
 *  - bf16 operands and outputs: conv1a's output, conv1b .. conv4b, convPa, convDa (ReLU in the epilogue), the 2x2
 *    max-pools, the inputs of convPb / convDb (whose outputs stay fp32), and in every GNN layer q|k|v, the attention
 *    message (mfr_superglue_attention: one fused launch, scores never stored), merge, mlp.0, and the input of mlp.3;
 *  - the token stream is fp32 with a bf16 shadow [x | message] refreshed after the keypoint encoder and after every
 *    layer's mlp.3 (which adds its output to the fp32 stream);
 *  - fp32 / tf32 as in MFR_PRECISION_TF32: the detector head and NMS, keypoint selection, descriptor normalisation and
 *    sampling, the keypoint encoder, final_proj, the score matrix, Sinkhorn and match extraction.
 * The "attn_scores" and "attn_vt" debug tensors do not exist in bf16 mode; "qkv" and "msg" hold bf16 there. */
int mfr_spsg_create_ex(int B, int H, int W, int max_keypoints, int nms_radius, float keypoint_threshold,
                       int remove_borders, int sinkhorn_iterations, float match_threshold, int precision,
                       mfr_spsg** out);
void mfr_spsg_destroy(mfr_spsg* h);
int mfr_spsg_num_weights(const mfr_spsg* h);
const char* mfr_spsg_weight_name(const mfr_spsg* h, int i);
long long mfr_spsg_weight_numel(const mfr_spsg* h, int i);
int mfr_spsg_set_weight(mfr_spsg* h, int i, const float* host, long long numel, void* stream);
int mfr_spsg_forward(mfr_spsg* h, const float* img0, const float* img1, void* stream);
/* Shared map frame: mfr_spsg_set_map runs SuperPoint once on the map image img0 [H][W] (device float32, eagerly) and
 * keeps its keypoints, scores and descriptors until the next set_map or weight upload; a paired mfr_spsg_forward in
 * between does not disturb them. mfr_spsg_forward_shared(h, img1 [B][H][W]) runs SuperPoint on the queries only, then
 * SuperGlue on every pair, and writes outputs bit-identical, in every precision, to mfr_spsg_forward(h, img0 repeated
 * B times, img1); it runs as its own CUDA graph and returns MFR_ERR_ARG before any set_map. */
int mfr_spsg_set_map(mfr_spsg* h, const float* img0, void* stream);
int mfr_spsg_forward_shared(mfr_spsg* h, const float* img1, void* stream);
void mfr_spsg_set_graph(mfr_spsg* h, int enabled);
int mfr_spsg_get_outputs(mfr_spsg* h, mfr_spsg_outputs* out);
int mfr_spsg_debug_tensor(mfr_spsg* h, const char* name, float** ptr, long long* numel);
int mfr_spsg_num_launches(const mfr_spsg* h);
/* SuperGlue alone (superglue.py:228-283) on caller-supplied SuperPoint outputs, HOST arrays in the
 * engine's layout: counts int[2B], keypoints float[2B][K][2], scores float[2B][K], descriptors
 * float[2B][K][256] (unused slots zero). Stage-boundary entry point. */
int mfr_spsg_forward_superglue(mfr_spsg* h, const int* counts, const float* keypoints, const float* scores,
                               const float* descriptors, void* stream);

/* Coarse matching on a materialised matrix (stage-boundary entry point of the LoFTR matcher):
 * CoarseMatching.forward dual-softmax + get_coarse_match of the reference
 * (LoFTR/src/loftr/utils/coarse_matching.py:109-119,175-196,242-259).
 *   sim: device float[B][L][L] similarity (already scaled by 1/(C*temperature)), or, when
 *   input_is_conf != 0, the confidence matrix itself (then the selection is bit-exact w.r.t. the
 *   reference's float-equality mutual-NN test on the same matrix).
 * Outputs (device, caller-owned): count int[1], offsets int[B+1], b/i/j_ids int[B*L],
 * mconf float[B*L], mkpts0_c/mkpts1_c float[B*L][2] = (idx % w_c, idx / w_c) * scale. */
int mfr_coarse_match(const float* sim, int B, int h_c, int w_c, float thr, int border_rm, float scale,
                     int input_is_conf, int* count, int* offsets, int* b_ids, int* i_ids, int* j_ids,
                     float* mconf, float* mkpts0_c, float* mkpts1_c, void* stream);

/* Exact 2-nearest-neighbour search (L2) of every query descriptor among the train descriptors:
 * the matcher of the reference's SIFT plugin (lib/models/matching/feature_matching.py:87-99),
 * knnMatch(k=2), as an exact brute-force search (the reference's FLANN kd-tree is approximate and
 * non-deterministic). query float[nq][dim], train float[nt][dim], dim % 4 == 0, dim <= 256 (device).
 * Outputs (device): idx1/idx2 int[nq] (-1 if absent), dist1/dist2 float[nq] (Euclidean). Ties go
 * to the lower index. */
int mfr_knn2_l2(const float* query, int nq, const float* train, int nt, int dim, int* idx1,
                float* dist1, int* idx2, float* dist2, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SIFT detector + descriptor engine. Replaces cv2.SIFT_create(nfeatures).detectAndCompute of the reference's SIFT
 * plugins (lib/models/matching/feature_matching.py:58,88-89, etc/feature_matching_baselines/matchers.py:158-161) at
 * OpenCV's default settings (3 layers per octave, contrast threshold 0.04, edge threshold 10, sigma 1.6, doubled
 * first octave, CV_32F descriptors), for B uint8 gray images [B][H][W] of one size per call (device memory).
 * nfeatures = 0: no cap; else retainBest(nfeatures): every keypoint whose response is >= the N-th largest (the
 * orientations of one point share a response, so an image may return more than N). max_candidates caps the refined
 * extrema and the oriented keypoints of an image; the true counts are reported, so the caller can detect an
 * overflow (results are then incomplete). root_sift != 0: descriptors are RootSIFT rows (L1 normalisation with
 * eps 1e-7, square root: feature_matching.py:67-73). Keypoints of an image are ordered by response descending, then
 * x, y, size, angle ascending. Deterministic: the same images give bit-identical outputs, whatever the batch. */
typedef struct mfr_sift mfr_sift;
typedef struct {
  const int* counts;          /* device int[B] keypoints per image */
  const int* raw_counts;      /* device int[B] oriented keypoints before duplicate removal / retainBest */
  const int* extrema_counts;  /* device int[B] refined extrema before orientation assignment */
  const float* keypoints;     /* device float[B][capacity][5]: x, y, size, angle, response (cv2.KeyPoint fields) */
  const int* octaves;         /* device int[B][capacity]: cv2.KeyPoint.octave (packed octave | layer << 8 | ...) */
  const float* descriptors;   /* device float[B][capacity][128] */
  int capacity;               /* = max_candidates */
} mfr_sift_outputs;
int mfr_sift_create(int B, int H, int W, int nfeatures, int max_candidates, int root_sift, mfr_sift** out);
void mfr_sift_destroy(mfr_sift* h);
/* imgs: device uint8 [B][H][W]. One static launch list (replayed as a CUDA graph unless disabled). */
int mfr_sift_detect(mfr_sift* h, const unsigned char* imgs, void* stream);
void mfr_sift_set_graph(mfr_sift* h, int enabled);
int mfr_sift_get_outputs(mfr_sift* h, mfr_sift_outputs* out);
/* Lowe ratio matching of the last detect for P = B / 2 pairs (images 2p, 2p + 1), the matcher of the SIFT plugins
 * (feature_matching.py:91-99, matchers.py:163-175) with an exact 2-NN (mfr_knn2_l2's search): query p's keypoint i
 * matches its nearest neighbour j in image 2p + 1 when d1 < ratio * d2 (and image 2p + 1 has >= 2 keypoints).
 * Matches are written in query order into caller-owned device buffers in the pose back end's layout:
 * kpts0 / kpts1 float[P * capacity][2] (x, y of keypoint i of image 2p / j of image 2p + 1), offsets int[P + 1]. */
int mfr_sift_match_pairs(mfr_sift* h, float ratio, float* kpts0, float* kpts1, int* offsets, void* stream);
/* named intermediate buffers for stage tests: "gauss_<o>" float[B][6][h_o][w_o], "dog_<o>" float[B][5][h_o][w_o]
 * (o = 0 is the doubled image), "kp_pre" float[B][capacity][5] / "kp_pre_octave" int[B][capacity] (oriented keypoints
 * before selection, internal octave coordinates, unordered), "counters" int[3][B] (extrema, oriented, selected) */
int mfr_sift_debug_tensor(mfr_sift* h, const char* name, float** ptr, long long* numel);
/* Eager detect with CUDA events between the stages: ms (host float[5]) = pyramid, extrema + refinement, orientation,
 * selection, descriptors. */
int mfr_sift_profile(mfr_sift* h, const unsigned char* imgs, float* ms, void* stream);

/* SIFT pair engine for P pairs of uint8 gray images [H][W]: detection (mfr_sift_detect's engine and settings) and Lowe ratio
 * matching (mfr_sift_match_pairs's) of both images of every pair, with the matches in engine-owned buffers in the pose
 * back end's layout. Bit-identical to mfr_sift_detect on the pair-interleaved batch (image 2p = img0[p], 2p + 1 =
 * img1[p]) followed by mfr_sift_match_pairs(ratio). Holds a B = 2P engine, a B = P engine for the queries of the shared
 * map path and a B = 1 engine for the map image. */
typedef struct mfr_sift_pairs mfr_sift_pairs;
typedef struct {
  const float* kpts0;         /* device float[capacity][2]: x, y of the matched keypoints of image 0, pair after pair */
  const float* kpts1;         /* device float[capacity][2]: their nearest neighbours in image 1 */
  const int* offsets;         /* device int[P + 1]: matches of pair p are rows offsets[p] .. offsets[p + 1] - 1 */
  const int* overflow;        /* device int[P]: 1 when an image of pair p (or the map) had more refined extrema or oriented
                                 keypoints than max_candidates; its matches are then incomplete */
  int capacity;               /* = P * max_candidates */
  int max_pts_per_pair;       /* = max_candidates: matches of one pair never exceed it */
} mfr_sift_pair_outputs;
int mfr_sift_pairs_create(int P, int H, int W, int nfeatures, int max_candidates, int root_sift, float ratio,
                          mfr_sift_pairs** out);
void mfr_sift_pairs_destroy(mfr_sift_pairs* h);
void mfr_sift_pairs_set_graph(mfr_sift_pairs* h, int enabled);
/* img0 / img1: device uint8 [P][H][W]. Two device copies stage them into the pair-interleaved input, then one launch list
 * (detect, 2-NN, ratio test, offsets, ordered compaction, overflow flags) runs as one CUDA graph. No host synchronisation
 * (after the first call, which captures the graph). Outputs are valid until the next forward on the handle. */
int mfr_sift_forward_pairs(mfr_sift_pairs* h, const unsigned char* img0, const unsigned char* img1, void* stream);
/* Detects and describes the map image img0 (device uint8 [H][W]) once, eagerly, into buffers of its own, valid until the
 * next set_map; paired forwards in between leave them intact. */
int mfr_sift_set_map(mfr_sift_pairs* h, const unsigned char* img0, void* stream);
/* img1: device uint8 [P][H][W] query images, ratio-matched against the map of set_map (the map's descriptors are the
 * knn query set, as image 0 of a pair is): the bits of mfr_sift_forward_pairs with the map repeated for every pair.
 * One CUDA graph; MFR_ERR_ARG before the first set_map. */
int mfr_sift_forward_shared(mfr_sift_pairs* h, const unsigned char* img1, void* stream);
int mfr_sift_get_pair_outputs(mfr_sift_pairs* h, mfr_sift_pair_outputs* out);

/* ---------------------------------------------------------------------------------------------
 * Pose back end (batched-hypothesis RANSAC). Replaces lib/models/matching/pose_solver.py.
 * Correspondences of P pairs are concatenated: kpts0/kpts1 device float[total][2] in pixels (x,y),
 * offsets device int[P+1]; K0/K1 device float[P][9] row-major intrinsics; depth maps device
 * float[P][H][W] metres (0 = invalid). Outputs: R float[P][9], t float[P][3], inliers int[P],
 * mask unsigned char[total]. Failure of a pair = NaN-filled R,t and 0 inliers
 * (pose_solver.py:30-33,50-51,146-150,189,198,231-233).
 * A solver handle owns the scratch memory; correspondences per pair are capped at 8192.       */
typedef struct mfr_pose_solver mfr_pose_solver;
int mfr_pose_solver_create(int max_pairs, int max_pts_per_pair, int max_hypotheses,
                           mfr_pose_solver** out);
void mfr_pose_solver_destroy(mfr_pose_solver* s);
/* Named scratch buffers of the handle, for stage-wise parity tests; *words is the buffer's size in 4-byte words. They
 * hold what the last call that wrote them left there:
 *   "hyp_results" block winners [max_pairs][*] {double cost; int count, valid; double model[12]} (112 bytes), row
 *                 stride = the blocks of that launch (E-mat: ceil(num_hyp / hypotheses per block); PnP: ceil(num_hyp / 128))
 *   "lo_results"  E-mat LO candidates [max_pairs][4] {double cost, R[9], t[3]} (104 bytes)
 *   "pts_norm"    float4 [max_pairs][max_pts_per_pair] normalised correspondences (x0, y0, x1, y1)
 *   "Rd", "td"    double [max_pairs][9] / [max_pairs][3]: the final E-mat pose
 *   "Xw", "uv", "vidx" PnP's compacted depth-valid points: double [max_pairs][max_pts_per_pair][3] (camera 0), float
 *                 [..][2] (kpts1), int [..] (index within the pair)
 *   "nvalid", "dmin" int [max_pairs] compacted count; float bits [max_pairs] of max(min(depth0), 0)
 *   "X1w", "dmin1" Procrustes: the compacted points lifted through depth1, double [max_pairs][max_pts_per_pair][3]
 *                 (camera 1; "Xw" holds their camera-0 partners); float bits [max_pairs] of max(min(depth1), 0)
 *   "icp_state"   double [max_pairs][18] of the last mfr_icp_refine: R [9], t [3] (source -> target), fitness, rmse,
 *                 stopped flag, correspondences of the last association, valid source / target points. A call with
 *                 max_iterations = k leaves the pose after k updates (fewer if it converged) and the association at
 *                 that pose. Exists after the first mfr_icp_refine call (MFR_ERR_ARG before). */
int mfr_pose_solver_debug_tensor(mfr_pose_solver* s, const char* name, void** ptr, long long* words);

/* EssentialMatrixSolver.estimate_pose (pose_solver.py:29-61): cv.findEssentialMat(USAC_MAGSAC) +
 * cv.recoverPose. `num_hyp` 5-point hypotheses per pair (MSAC-scored). lo_enabled is a bit set:
 *   bit 0 (1): local optimisation of the 4 best block winners (LM on a Tukey M-estimator of the Sampson distance,
 *              cut-off 3x -> 1x the threshold) + noise-adaptive tightening;
 *   bit 1 (2): final truncated least-squares refit at the threshold (LM on the MSAC cost): the result is the Sampson
 *              least-squares optimum of its OWN inlier set — the point the reference's output polished by LM on its
 *              own mask sits at (SURVEY §7 hard part 1(b)); needs bit 0.
 * t has unit norm; max_pts_per_pair <= 8192 (more correspondences of a pair are ignored). The final (R, t) is also
 * kept in fp64 inside the handle for mfr_scale_from_depth. */
int mfr_emat_ransac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets,
                    int P, const float* K0, const float* K1, float pix_threshold, int num_hyp,
                    unsigned long long seed, int lo_enabled, float* R, float* t, int* n_inliers,
                    unsigned char* mask, void* stream);

/* EssentialMatrixMetricSolver.estimate_pose (pose_solver.py:132-172), the part after the
 * scale-free solve: depth lookup at int-truncated inlier keypoints, back-projection, per-point
 * scale, exhaustive consensus with |s - s_hyp| < scale_threshold. Rd/td: device double[P][9]/[P][3]
 * pose to use, or NULL to take the pose left in the handle by mfr_emat_ransac. */
int mfr_scale_from_depth(mfr_pose_solver* s, const float* kpts0, const float* kpts1,
                         const int* offsets, int P, const float* K0, const float* K1,
                         const unsigned char* mask, const double* Rd, const double* td,
                         const float* depth0, const float* depth1, int H, int W,
                         float scale_threshold, float* R_out, float* t_metric, int* inliers,
                         void* stream);

/* PnPSolver.estimate_pose (pose_solver.py:184-235): lift kpts0 through depth0 (valid iff depth >
 * depth0.min()), P3P RANSAC on (xyz0, kpts1) with reprojection threshold in pixels, LM refinement
 * on the inliers when there are >= 6, reject |t| > 1000. */
int mfr_pnp_ransac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets,
                   int P, const float* K0, const float* K1, const float* depth0, int H, int W,
                   int num_hyp, float reproj_threshold, unsigned long long seed, float* R, float* t,
                   int* n_inliers, unsigned char* mask, void* stream);

/* mfr_emat_ransac / mfr_pnp_ransac with the CONFIDENCE escalation of the solver plugins (pose_solver._SolverBase:
 * EMAT_RANSAC.CONFIDENCE / PNP.CONFIDENCE up to GPU_RANSAC.MAX_HYPOTHESES), per pair, on the device:
 *   budgets  h0 = num_hyp, then min(max_hyp, 4 h_prev) while h_prev < max_hyp. Every round is enqueued up front; a round
 *            is the fixed-budget call at its budget (same seed, same block partition) restricted to the pairs still
 *            active, and a pair that is done skips the later rounds' blocks. No host synchronisation: the call can be
 *            captured in a CUDA graph.
 *   rule     after the round at h, a pair stops iff h >= required(confidence, n / N, s) with N = min(offsets[p+1] -
 *            offsets[p], max_pts_per_pair), n its inliers at h, s = 5 (E-mat) or 4 (PnP), required = the number of
 *            samples after which an all-inlier sample has been drawn with probability confidence (capped at 2^31 - 1).
 *            n <= 0 stops only at max_hyp (the NaN pose stands). A pair with N < s is done after round 0 with budget 0.
 *   result   pair p's outputs (R, t, n_inliers, its mask rows; for E-mat also the fp64 pose kept for
 *            mfr_scale_from_depth) equal bit for bit those of the fixed-budget call on the same batch at num_hyp =
 *            budgets_out[p], the budget at which it stopped (max_hyp if it never did).
 * budgets_out: device int[P], or NULL. confidence <= 0: one round at num_hyp. num_hyp < 1, max_hyp < num_hyp or max_hyp
 * above the handle's max_hypotheses: MFR_ERR_ARG (nothing is clipped).
 * The rule is evaluated with the device's fp64 log / log1p / pow, which may differ from the host libm's in the last bit:
 * a decision can differ from the plugins' only where the required count lies within ~1e-15 (relative) of a budget. */
int mfr_emat_ransac_escalate(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets,
                             int P, const float* K0, const float* K1, float pix_threshold, int num_hyp,
                             unsigned long long seed, int lo_enabled, float* R, float* t, int* n_inliers,
                             unsigned char* mask, double confidence, int max_hyp, int* budgets_out, void* stream);
int mfr_pnp_ransac_escalate(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets,
                            int P, const float* K0, const float* K1, const float* depth0, int H, int W,
                            int num_hyp, float reproj_threshold, unsigned long long seed, float* R, float* t,
                            int* n_inliers, unsigned char* mask, double confidence, int max_hyp, int* budgets_out,
                            void* stream);

/* mfr_emat_ransac_escalate with the estimator of the reference's cv.USAC_MAGSAC: MAGSAC++ (Barath et al., CVPR 2020)
 * in place of MSAC and its LO. Same arguments without lo_enabled.
 *   loss     rho of the Sampson distance r (normalised coordinates) for nu = 4 degrees of freedom, sigma_max = the
 *            normalised threshold pix_threshold / mean(K0.fx, K1.fy, K0.fy, K1.fx), cut-off k sigma_max with k = 3.64
 *            (mfr_host_magsac_loss evaluates it).
 *   scoring  each 5-point hypothesis scores sum rho (fp32 per point); the inlier count at the threshold is unchanged.
 *   LO       sigma-consensus++ (IRLS / LM on sum rho in fp64, MAGSAC++ weights) from each of the 4 cheapest block
 *            winners, at most 10 passes over a strided subsample of <= 1024 correspondences; the candidate with the
 *            lowest sum rho over all correspondences is polished the same way on all of them, at most 30 passes.
 *            Both stop once sum rho drops by <= 1e-10 (relative). No noise-adaptive tightening, no least-squares refit.
 *   outputs  as mfr_emat_ransac: mask = Sampson^2 < threshold^2 under the final E, filtered by recoverPose's
 *            cheirality vote; the fp64 pose is kept for mfr_scale_from_depth. "hyp_results" / "lo_results" hold sum rho
 *            as their costs.
 * confidence <= 0: one round at num_hyp (max_hyp must still be >= num_hyp); otherwise the escalation contract of
 * mfr_emat_ransac_escalate, with the same budget sequence, rule and bit-for-bit result. Capturable in a CUDA graph. */
int mfr_emat_magsac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets, int P,
                    const float* K0, const float* K1, float pix_threshold, int num_hyp, unsigned long long seed,
                    float* R, float* t, int* n_inliers, unsigned char* mask, double confidence, int max_hyp,
                    int* budgets_out, void* stream);

/* ProcrustesSolver.estimate_pose with REFINE = False (pose_solver.py:247-320): lift both keypoint sets
 * through their depth maps (valid iff depth > depth.min() on both sides), RANSAC over 3-point Kabsch
 * alignments with inlier distance max_corr_dist (metres), refit on the inliers. The reference calls
 * Open3D's registration_ransac_based_on_correspondence for this step; REFINE = True continues with mfr_icp_refine. */
int mfr_procrustes_ransac(mfr_pose_solver* s, const float* kpts0, const float* kpts1, const int* offsets,
                          int P, const float* K0, const float* K1, const float* depth0,
                          const float* depth1, int H, int W, int num_hyp, float max_corr_dist,
                          unsigned long long seed, float* R, float* t, int* n_inliers, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Host test hooks: the minimal solvers used inside the RANSAC kernels are __host__ __device__
 * functions; these run the very same code on the CPU so that it can be unit-tested without a GPU.
 * They are NOT a CPU fallback: no product entry point calls them.
 *   five_point : x0, x1 double[5][2] normalised points, E_out double[10][9]; returns #solutions
 *   p3p        : X double[3][3] points, f double[3][3] unit bearings, R_out [4][9], t_out [4][3]
 *   kabsch     : the least-squares rigid transform of the Procrustes / ICP kernels (q ~ R p + t) from the moment sums
 *                n, sum_p [3], sum_q [3], sum_pq [9] (row-major sum p q^T); R_out [9], t_out [3]; returns 1, or 0 when
 *                n < 3 or the points are coincident or collinear
 *   poly roots : coef[0..deg] ascending, deg <= 10; returns #real roots (ascending)
 *   ransac_satisfied : 1 iff the escalation stops after a round at `budget` that found n_inliers of n_points
 *                (the rule of mfr_emat_ransac_escalate, cap max_budget, minimal sample sample_size), else 0
 *   magsac_loss : MAGSAC++ rho(r) and w(r) = rho'(r) / r of mfr_emat_magsac (the fp64 version of its LO / polish) for
 *                a Sampson distance r and sigma_max > 0 (else MFR_ERR_ARG)
 *   jpeg_decode : mfr_jpeg_decode's arithmetic run serially on the CPU; data and dst in HOST memory, dst sized
 *                width x height (x 3 when rgb), the oriented size; returns the file's status
 *   png_decode : mfr_png_decode_batch's arithmetic for one file run serially on the CPU; data and dst in HOST memory,
 *                dst sized width x height samples of the out_kind's type (mfr_png_info's size); returns the file's
 *                status                                                                                         */
int mfr_host_five_point(const double* x0, const double* x1, double* E_out);
int mfr_host_p3p(const double* X, const double* f, double* R_out, double* t_out);
int mfr_host_kabsch(double n, const double* sum_p, const double* sum_q, const double* sum_pq, double* R_out,
                    double* t_out);
int mfr_host_poly_real_roots(const double* coef, int deg, double* roots);
int mfr_host_decompose_essential(const double* E, double* R1, double* R2, double* t);
int mfr_host_ransac_satisfied(double confidence, int n_inliers, int n_points, int budget, int max_budget,
                              int sample_size);
int mfr_host_magsac_loss(double r, double sigma_max, double* rho, double* w);
int mfr_host_jpeg_decode(const unsigned char* data, long long length, int rgb, unsigned char* dst, int width, int height);
int mfr_host_png_decode(const unsigned char* data, long long length, int out_kind, void* dst, int width, int height);

/* Debug probe (scripts/png_decode_bench.py): milliseconds of the CRC, inflate and unfilter kernels (ms[0..2], CUDA
 * events) of the decoder's last mfr_png_decode_batch call; waits for that call's kernels. */
typedef struct mfr_png_decoder mfr_png_decoder;
int mfr_debug_png_kernel_ms(mfr_png_decoder* dec, float* ms);

/* Debug probe (microbenchmark used by scripts/, not part of the product path): microseconds per
 * launch of a prebuilt conv/GEMM op launched back to back.
 * flags: bit 0 = x/w are bf16, bit 1 = out/residual are bf16, bit 2 = channel strides padded to multiples of 8 elements;
 * residual may be NULL */
float mfr_debug_time_conv(const float* x, int N, int H, int W, int Cin, const float* w, int Cout, int R,
                          int stride, float* out, int iters, int flags, const float* residual);

/* Stage entry for tests: LoFTR's linear attention (LoFTR/src/loftr/loftr_module/linear_attention.py:31-45) on
 * already feature-mapped q' = elu(q)+1, k' and values. windows = 0: q [n][L][256], k / v [n][S][256], 8 heads of 32
 * (coarse level); windows = 1: q, k, v [n][25][128], 8 heads of 16, n items (fine level, L and S ignored).
 * bf16 = 0: fp32 tensors, q and k already feature-mapped. bf16 = 2: bf16 tensors (the tensor-core kernels) with RAW q and k
 * (the projections as the GEMM leaves them): the kernels apply elu(x) + 1 themselves. bf16 = 1 (bf16 tensors with
 * pre-mapped q, k) returns MFR_ERR_UNSUPPORTED. Device pointers, dense rows. */
int mfr_linear_attention(const void* q, const void* k, const void* v, void* msg, int n, int L, int S, int windows,
                         int bf16, void* stream);

/* Stage entry for tests: SuperGlue's multi-head softmax attention (SuperGlue/models/superglue.py:85-89), the fused
 * kernel of the bf16 engine mode. qkv: device bf16 [n_img][max_kp][ldq], columns q | k | v (0-255, 256-511, 512-767;
 * head h at 64 h), counts: device int[n_img]. Image i attends to the first counts[i ^ cross] keys / values of image
 * i ^ cross (cross 0 or 1; images pair-interleaved). msg: device bf16 [n_img][max_kp][ldo], channel 64 h + d;
 * rows >= counts[i], and every row when counts[i ^ cross] == 0, are written as zeros. max_kp: multiple of 16 in
 * [16, 2048]; ldq >= 768 and a multiple of 8, ldo >= 256 and even; qkv 16-byte aligned. */
int mfr_superglue_attention(const void* qkv, long long ldq, const int* counts, int n_img, int max_kp, int cross,
                            void* msg, long long ldo, void* stream);

/* Stage entry for tests: the backbone stem, conv 7x7 stride 2 pad 3, 1 -> 128 channels, folded-BN bias, ReLU
 * (LoFTR/src/loftr/backbone/resnet_fpn.py:52-62,102). img fp32 [NI][H][W]; w fp32 [128][49]; out [NI][H/2][W/2][128], bf16 when
 * out_bf16 != 0, else fp32 (both on mma.sync); exact_fp32: plain FMA kernel. */
int mfr_stem_conv7x7(const float* img, const float* w, const float* bias, void* out, int NI, int H, int W, int out_bf16,
                     int exact_fp32, void* stream);

/* ProcrustesSolver's ICP refinement (PROCRUSTES.REFINE, pose_solver.py:289-315: Open3D registration_icp, point-to-point,
 * correspondence radius max_corr_dist, criteria relative_fitness / relative_rmse / max_iterations = 1e-4 / 1e-4 / 30 in the
 * reference) of the poses (R_in, t_in) [P][9] / [P][3] over the FULL clouds of both depth maps (every pixel with depth > 0),
 * device float [P][H][W]. Nearest neighbours are exact within the radius (window search in the organised target cloud,
 * clamped to 96 pixels and widened when a nearer point could lie beyond the clamp) for every target point at least
 * 2 max_corr_dist + 1 mm in front of camera 1. The per-pass sums are added in a fixed order over chunks of the frame, so a
 * pair's result is bit for bit the same alone, in any batch, on any GPU and in a graph replay. The first call at a
 * larger H x W allocates scratch: make it before capturing the call in a CUDA graph.
 * n_inliers = int(fitness * valid target points), the reference's return value (pose_solver.py:319). */
int mfr_icp_refine(mfr_pose_solver* s, const float* depth0, const float* depth1, int H, int W, int P, const float* K0,
                   const float* K1, const float* R_in, const float* t_in, float max_corr_dist, int max_iterations,
                   float relative_fitness, float relative_rmse, float* R, float* t, int* n_inliers, void* stream);

/* Input path on the GPU (SURVEY §8(f) rank 1): JPEG decode with cv2.imread's exact pixels, and cv2.resize.
 *
 * JPEG decode (csrc/jpeg.cuh, csrc/image_io.cu): libjpeg(-turbo)'s decompression arithmetic as CUDA kernels (ISLOW IDCT,
 * fancy upsampling, its YCbCr -> RGB tables) plus the Exif Orientation that cv2.imread applies. Output in DEVICE memory:
 * rgb = 0: gray [h][w], the Y plane as coded (cv2.imread(IMREAD_GRAYSCALE), SuperGlue/models/utils.py:264); rgb = 1:
 * interleaved RGB [h][w][3] (cv2.imread(IMREAD_COLOR) in RGB order, lib/datasets/utils.py:67); h, w after the
 * orientation (5-8 swap them). Supported: SOF0 / SOF1 8-bit Huffman, one interleaved scan, gray or YCbCr with luma
 * sampling 1x1 / 2x1 / 2x2 and chroma 1x1, any size, DRI / RSTn, 8- or 16-bit quantisation tables. A valid file outside
 * that set gives MFR_ERR_UNSUPPORTED (progressive, arithmetic, lossless, 12-bit, 4:4:0, 4:1:1, CMYK, RGB-coded,
 * multi-scan); malformed headers give MFR_ERR_ARG; entropy-coded data with an invalid code, or that ends before its
 * last block, gives MFR_ERR_ARG once decoded (libjpeg decodes such data with warnings: cv2 is the answer for it).
 *   mfr_jpeg_info: parses one file (HOST bytes): oriented width / height and component count, or the file's error code.
 *   mfr_jpeg_decode: one file through a process-wide decoder per device (created on first use, grown when a file does
 *     not fit, guarded by a mutex); width / height must be mfr_jpeg_info's. Returns once the image is decoded, with its
 *     status.
 *   mfr_jpeg_decoder_create: a decoder for batches of up to max_images files holding up to max_bytes of entropy-coded
 *     data and max_pixels pixels in all, each image counted at its size rounded up to multiples of 16 (what its
 *     coefficient planes need). It owns pinned staging, device buffers and two events; not thread-safe.
 *   mfr_jpeg_batch_info: per file (HOST arrays) the oriented width / height (0 unless supported) and status MFR_OK,
 *     MFR_ERR_UNSUPPORTED or MFR_ERR_ARG, from the headers alone.
 *   mfr_jpeg_decode_batch: decodes n files (HOST byte pointers and lengths) into dst[i] (DEVICE pointers, sized from
 *     mfr_jpeg_batch_info; ignored for files that are not MFR_OK there) asynchronously on `stream`: it returns once the
 *     work is enqueued, the bytes having been copied into the decoder's staging. status: DEVICE int[n], written on the
 *     stream: the header status of each file, then MFR_ERR_ARG where its entropy-coded data fails. The call returns
 *     MFR_ERR_ARG when the batch exceeds the decoder's capacity (nothing is enqueued). Successive calls on one decoder
 *     may use different streams: each waits on the device for the previous call's kernels.
 * mfr_resize_linear: cv2.resize(INTER_LINEAR) + scale on the device, dst fp32 [dst_h][dst_w][channels] (chw = 0) or
 * [channels][dst_h][dst_w] (chw = 1) = resized * out_scale. mode 0: float source, float arithmetic; mode 1: uint8 source
 * converted to float first (read_image with resize_float = True, utils.py:272-273: the FMB matcher plugins);
 * mode 2: uint8 source, OpenCV's 11-bit fixed-point uint8 path, rounded to uint8 before the scale (utils.py:275,
 * lib/datasets/utils.py:68). src_row_stride in elements. */
typedef struct mfr_jpeg_decoder mfr_jpeg_decoder;
int mfr_jpeg_info(const unsigned char* data, long long length, int* width, int* height, int* components);
int mfr_jpeg_decode(const unsigned char* data, long long length, int rgb, unsigned char* dst, int width, int height, void* stream);
int mfr_jpeg_decoder_create(int max_images, long long max_bytes, long long max_pixels, mfr_jpeg_decoder** out);
void mfr_jpeg_decoder_destroy(mfr_jpeg_decoder* dec);
int mfr_jpeg_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* status);
int mfr_jpeg_decode_batch(mfr_jpeg_decoder* dec, const unsigned char* const* data, const long long* lengths, int n, int rgb,
                          unsigned char* const* dst, int* status, void* stream);

/* 16-bit depth PNG decode on the GPU (lib/datasets/utils.py:77-81, read_depth_image: cv2.imread(path, IMREAD_UNCHANGED)
 * / 1000, then .float()). Supported: non-interlaced gray PNGs (colour type 0) of bit depth 8 or 16, any size within
 * libpng's default limits and OpenCV's, any IDAT chunking and any deflate content, with only tEXt / zTXt / iTXt / tIME /
 * pHYs besides the critical chunks. A valid file outside that set gives MFR_ERR_UNSUPPORTED (other colour types and
 * depths, Adam7, PLTE / tRNS / sBIT / gAMA / iCCP / eXIf / APNG and unknown chunks); malformed structure gives
 * MFR_ERR_ARG (signature, chunk lengths, IHDR fields, chunk order, a missing IEND, the zlib header, the CRC of IHDR or
 * IEND). On the device, a file whose IDAT CRC, deflate data, Adler-32 or row filter types fail gets MFR_ERR_ARG: libpng
 * refuses such files, so a caller that falls back to cv2 for it gets cv2's answer.
 *   mfr_png_info: parses one file (HOST bytes): width, height, bit depth, or the file's error code.
 *   mfr_png_decoder_create: a decoder for batches of up to max_images files holding up to max_bytes of zlib data and
 *     max_pixels pixels in all. It owns pinned staging, device buffers and two events; not thread-safe.
 *   mfr_png_batch_info: per file (HOST arrays) width / height / bit depth (0 unless supported) and status MFR_OK,
 *     MFR_ERR_UNSUPPORTED or MFR_ERR_ARG, from the chunk structure alone.
 *   mfr_png_decode_batch: decodes n files (HOST byte pointers and lengths) into dst[i] (DEVICE pointers; ignored for
 *     files that are not MFR_OK in mfr_png_batch_info) asynchronously on `stream`; the bytes are copied into the
 *     decoder's staging before it returns. out_kind 0: the samples as stored, uint8 or uint16 (native order) [h][w] =
 *     cv2.imread(IMREAD_UNCHANGED); out_kind 1: float32 [h][w] = (float)((double)v / 1000). status: DEVICE int[n],
 *     written on the stream: the header status of each file, then MFR_ERR_ARG where its data fails a device check.
 *     MFR_ERR_ARG when the batch exceeds the decoder's capacity (nothing is enqueued). Successive calls on one decoder
 *     may use different streams: each waits on the device for the previous call's kernels. */
int mfr_png_info(const unsigned char* data, long long length, int* width, int* height, int* bit_depth);
int mfr_png_decoder_create(int max_images, long long max_bytes, long long max_pixels, mfr_png_decoder** out);
void mfr_png_decoder_destroy(mfr_png_decoder* dec);
int mfr_png_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* bit_depth,
                       int* status);
int mfr_png_decode_batch(mfr_png_decoder* dec, const unsigned char* const* data, const long long* lengths, int n, int out_kind,
                         void* const* dst, int* status, void* stream);
int mfr_resize_linear(const void* src, int src_is_u8, int src_w, int src_h, long long src_row_stride, int channels, float* dst,
                      int dst_w, int dst_h, int mode, float out_scale, int chw, void* stream);

/* Leaderboard metrics of the Map-free benchmark for n poses (benchmark/metrics.py:40-67, benchmark/utils.py:95-129 sine
 * variant, benchmark/reprojection.py:7-86): device double arrays q_gt/q_est [n][4] (w, x, y, z), t_gt/t_est [n][3],
 * K [n][9]; image size W x H. Out: trans_err [n] (m), rot_err [n] (degrees), reproj_err [n] (VCRE, pixels). */
int mfr_pose_metrics(const double* q_gt, const double* t_gt, const double* q_est, const double* t_est, const double* K, int W,
                     int H, int n, double* trans_err, double* rot_err, double* reproj_err, void* stream);

/* Stage entry: the tail of one LoFTREncoderLayer (loftr_module/transformer.py:52-58),
 *   x += norm2(mlp2(relu(mlp0([x | norm1(merge(msg))])))),  bf16 tensor-core operands, fp32 accumulate / LayerNorm / residual,
 * for n_blocks row blocks of rows_cap token rows (live rows per block: *dyn_rows when non-null). Device pointers:
 * msg bf16 [rows][C]; xb bf16 [rows][2C] (columns [0, C) = shadow of x: read, then rewritten with the new x);
 * x fp32 [rows][2C] (columns [0, C) in / out); w_merge [C][C], w_mlp0 [2C][2C], w_mlp2 [C][2C] bf16 row-major
 * ([out][in], the reference's nn.Linear layout); g1 / b1 / g2 / b2 fp32 [C]. C = 256 or 128. One fused wgmma kernel
 * launch (csrc/encoder_tail.cu, the engine's bf16 path). `iters` launches back to back (timing); note that every launch
 * applies the residual update again. */
int mfr_encoder_tail(const void* msg, void* xb, float* x, const void* w_merge, const void* w_mlp0, const void* w_mlp2,
                     const float* g1, const float* b1, const float* g2, const float* b2, int C, int n_blocks,
                     long long rows_cap, const int* dyn_rows, int iters, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MFR_B200_H_ */
