// SuperPoint + SuperGlue matcher engine (B image pairs per call): static launch list of wgmma
// conv/GEMM launches + SIMT kernels, replayed through a CUDA graph. Mirrors the reference's
// SuperGlue/models/matching.py:56-84 (SuperPoint x2 -> SuperGlue) with the settings hard-wired in
// etc/feature_matching_baselines/matchers.py:65-71 (nms 4, threshold 0.005, <= 1024 keypoints,
// 20 Sinkhorn iterations, match threshold 0.2). Images are stored pair-interleaved
// (image 2p = pair p's image0, 2p+1 = image1) so that the cross-attention partner is `img ^ 1`.
#include "spsg_engine.cuh"

#include <string>

#include "conv_gemm.cuh"
#include "engine_core.cuh"
#include "loftr_ops.cuh"   // rows_split3 (3xTF32 operand split of the fp32-faithful mode), rows_to_bf16
#include "sg_attention.cuh"
#include "spsg_ops.cuh"

namespace mfr {

struct SpsgEngine : EngineCore {
  int B, H, W, NI, K;  // K = max keypoints per image
  float kp_thr, match_thr;
  int nms_r, border, sk_iters;
  float bin_score = 1.f;
  long long bin_gen = -1;   // weight generation bin_score was read from
  size_t sg_begin = 0;   // first step of the SuperGlue part
  // Shared map frame (set_map / forward_shared): map_steps runs SuperPoint on one image into the map_* buffers;
  // shared_steps runs it on the B queries into the q_* buffers, interleaves map and queries into the pair layout and
  // continues with the paired list's SuperGlue steps.
  LaunchList map_steps, shared_steps;
  GraphExec graph, shared_graph;
  int *map_counts = nullptr, *q_counts = nullptr;
  float *map_kpts = nullptr, *map_kscores = nullptr, *map_D = nullptr, *q_kpts = nullptr, *q_kscores = nullptr, *q_D = nullptr;
  long long map_gen = -1;   // weight generation the map was encoded with (-1: no map)
  // buffers
  float* img;
  float *kpts, *kscores, *X, *D, *mk0, *mk1, *mscores0;
  int *counts, *matches0, *m_offsets;
  // precision 2 (fp32-faithful, MFR_PRECISION_FP32X3): every tensor-core GEMM runs as a 3xTF32 split product over 3x the
  // K extent; A operands are split [hi | lo | hi] into the scratch x3 right before the GEMM, weights [hi | hi | lo] into
  // `derived` once per upload (see loftr_ops.cu: rows_split3)
  // precision 1 (MFR_PRECISION_BF16): `derived` holds bf16 copies of the GEMM weights (every bf16 GEMM has a Cin that
  // is a multiple of 8, so rows need no padding), converted once per upload
  int precision = 0;
  float* x3 = nullptr; size_t x3_cap = 0;
  DerivedWeights derived{&rc};

  void push(std::function<int(cudaStream_t)> f, int n_launch = 1) { steps.push(std::move(f), "", n_launch); }

  void gemm(const std::string& w, const float* x, int N, int Hh, int Ww, int Cin, long long ldx, int Cout, int R,
            int act, const float* residual, float* out, long long ldo, long long ldr = 0, int in_bf16 = 0,
            int out_bf16 = 0) {
    ConvGemmDesc d{};
    d.x = x; d.N = N; d.H = Hh; d.W = Ww; d.Cin = Cin; d.ldx = ldx;
    d.w = weights[w + ".w"];
    if (in_bf16) {   // bf16 x and weights (ldw = Cin); out / residual bf16 when out_bf16
      d.in_bf16 = 1; d.out_bf16 = out_bf16;
      d.w = derived.get(weights, w + ".w", static_cast<long long>(Cout) * R * R, Cin);
    }
    if (precision == 2) {
      const long long rows_img = static_cast<long long>(Hh) * Ww;
      if (static_cast<size_t>(N) * rows_img * 3 * Cin > x3_cap || (Cin & 3)) { rc = MFR_ERR_ARG; return; }
      float* x3_ = x3; const int N_ = N, C_ = Cin;
      push([=](cudaStream_t st) { return rows_split3(x, ldx, rows_img * ldx, x3_, rows_img, N_, C_, 0, nullptr, st); });
      d.x = x3; d.Cin = 3 * Cin; d.ldx = 3 * Cin;
      d.w = derived.get(weights, w + ".w", static_cast<long long>(Cout) * R * R, Cin);
    }
    d.Cout = Cout; d.R = R; d.S = R; d.stride = 1; d.pad = R / 2;
    d.bias = weights[w + ".b"]; d.residual = residual; d.ldr = ldr > 0 ? ldr : ldo; d.act = act; d.alpha = 1.f; d.out = out; d.ldo = ldo;
    ConvGemmParams p;
    int r = conv_gemm_build(d, &p);
    if (r != MFR_OK) { rc = r; return; }
    push([p](cudaStream_t st) { return conv_gemm_launch(p, st); });
  }

  int build() {
    NI = 2 * B;
    // ---- weight table
    weights.add("conv1a.w", 64 * 9); weights.add("conv1a.b", 64);
    auto cv = [&](const std::string& n, int ci, int co, int r) {
      weights.add(n + ".w", static_cast<size_t>(co) * r * r * ci);
      weights.add(n + ".b", co);
    };
    cv("conv1b", 64, 64, 3); cv("conv2a", 64, 64, 3); cv("conv2b", 64, 64, 3); cv("conv3a", 64, 128, 3);
    cv("conv3b", 128, 128, 3); cv("conv4a", 128, 128, 3); cv("conv4b", 128, 128, 3);
    cv("convPa", 128, 256, 3); cv("convPb", 256, 65, 1); cv("convDa", 128, 256, 3); cv("convDb", 256, 256, 1);
    cv("kenc.0", 4, 32, 1); cv("kenc.1", 32, 64, 1); cv("kenc.2", 64, 128, 1); cv("kenc.3", 128, 256, 1); cv("kenc.4", 256, 256, 1);
    for (int i = 0; i < 18; ++i) {
      const std::string p = "gnn." + std::to_string(i);
      cv(p + ".qkv", 256, 768, 1); cv(p + ".merge", 256, 256, 1); cv(p + ".mlp0", 512, 512, 1); cv(p + ".mlp3", 512, 256, 1);
    }
    cv("final_proj", 256, 256, 1);
    weights.add("bin_score", 1);
    weights.alloc(mem);
    const bool bf = precision == 1;
    if (bf) derived.alloc(mem, weights, DerivedWeights::kBf16);
    if (precision == 2) {
      derived.alloc(mem, weights, DerivedWeights::kSplit3);
      const size_t act = static_cast<size_t>(2) * B * H * W * 64;                         // largest conv input (conv1b)
      const size_t att = static_cast<size_t>(2) * B * (4 * static_cast<size_t>(K) * K + 256 * static_cast<size_t>(K));   // P + V^T
      x3_cap = 3 * std::max(act, std::max(att, static_cast<size_t>(2) * B * K * 768));
      x3 = mem.alloc<float>(x3_cap, "split3_scratch");
    }

    const int H2 = H / 2, W2 = W / 2, H4 = H2 / 2, W4 = W2 / 2, h8 = H4 / 2, w8 = W4 / 2;
    const int Hs = h8 * 8, Ws = w8 * 8;
    auto px = [&](int hh, int ww) { return static_cast<size_t>(NI) * hh * ww; };
    img = mem.alloc<float>(px(H, W), "img");
    // SuperPoint activations up to the heads' inputs: bf16 storage in bf16 mode (float-typed pointers)
    auto act = [&](size_t n, const char* name = nullptr) {
      return bf ? reinterpret_cast<float*>(mem.alloc<unsigned short>(n, name)) : mem.alloc<float>(n, name);
    };
    float* x1a = act(px(H, W) * 64, "x1a"); float* x1b = act(px(H, W) * 64);
    float* p1 = act(px(H2, W2) * 64); float* x2a = act(px(H2, W2) * 64); float* x2b = act(px(H2, W2) * 64);
    float* p2 = act(px(H4, W4) * 64); float* x3a = act(px(H4, W4) * 128); float* x3b = act(px(H4, W4) * 128);
    float* p3 = act(px(h8, w8) * 128); float* x4a = act(px(h8, w8) * 128); float* x4b = act(px(h8, w8) * 128, "x4b");
    float* cPa = act(px(h8, w8) * 256, "cPa"); float* logits = mem.alloc<float>(px(h8, w8) * 65, "logits");
    float* scores = mem.alloc<float>(px(Hs, Ws), "scores"); float* mask = mem.alloc<float>(px(Hs, Ws), "nms_mask");
    float* t0 = mem.alloc<float>(px(Hs, Ws)); float* t1 = mem.alloc<float>(px(Hs, Ws)); float* t2 = mem.alloc<float>(px(Hs, Ws)); float* t3 = mem.alloc<float>(px(Hs, Ws));
    float* cDa = act(px(h8, w8) * 256, "cDa"); float* dense = mem.alloc<float>(px(h8, w8) * 256, "dense_desc");
    kpts = mem.alloc<float>(static_cast<size_t>(NI) * K * 2, "keypoints"); kscores = mem.alloc<float>(static_cast<size_t>(NI) * K, "kscores");
    counts = mem.alloc<int>(NI);
    X = mem.alloc<float>(static_cast<size_t>(NI) * K * 512, "tokens");
    D = mem.alloc<float>(static_cast<size_t>(NI) * K * 256, "descriptors");
    const size_t rows = static_cast<size_t>(NI) * K;
    float* kin = mem.alloc<float>(rows * 4); float* k1 = mem.alloc<float>(rows * 32); float* k2 = mem.alloc<float>(rows * 64);
    float* k3 = mem.alloc<float>(rows * 128); float* k4 = mem.alloc<float>(rows * 256);
    float *qkv = nullptr, *msg = nullptr, *h1 = nullptr, *Xb = nullptr, *Sat = nullptr, *Vt = nullptr;
    if (!bf) {
      qkv = mem.alloc<float>(rows * 768, "qkv"); msg = mem.alloc<float>(rows * 256, "msg"); h1 = mem.alloc<float>(rows * 512);
    } else {   // bf16 storage: q|k|v, the attention message, the hidden layer, and the token shadow [x | message]
      qkv = reinterpret_cast<float*>(mem.alloc<unsigned short>(rows * 768, "qkv"));
      msg = reinterpret_cast<float*>(mem.alloc<unsigned short>(rows * 256, "msg"));
      h1 = reinterpret_cast<float*>(mem.alloc<unsigned short>(rows * 512));
      Xb = reinterpret_cast<float*>(mem.alloc<unsigned short>(rows * 512, "tokens_bf16"));
    }
    float* Mb = mem.alloc<float>(rows * 256, "mdesc");
    if (!bf) {   // tensor-core attention: scores / probabilities [NI][4 heads][K][K] and V transposed [NI][256][K]
      Sat = mem.alloc<float>(static_cast<size_t>(NI) * 4 * K * K, "attn_scores");
      Vt = mem.alloc<float>(static_cast<size_t>(NI) * 256 * K, "attn_vt");
    }
    float* S = mem.alloc<float>(static_cast<size_t>(B) * K * K, "sg_scores");
    float* u = mem.alloc<float>(static_cast<size_t>(B) * (K + 1), "sk_u"); float* v = mem.alloc<float>(static_cast<size_t>(B) * (K + 1), "sk_v");
    float* rmax = mem.alloc<float>(static_cast<size_t>(B) * K); int* rarg = mem.alloc<int>(static_cast<size_t>(B) * K); int* carg = mem.alloc<int>(static_cast<size_t>(B) * K);
    matches0 = mem.alloc<int>(static_cast<size_t>(B) * K); mscores0 = mem.alloc<float>(static_cast<size_t>(B) * K, "mscores0");
    mk0 = mem.alloc<float>(static_cast<size_t>(B) * K * 2); mk1 = mem.alloc<float>(static_cast<size_t>(B) * K * 2);
    m_offsets = mem.alloc<int>(B + 1);
    map_counts = mem.alloc<int>(1); q_counts = mem.alloc<int>(B);
    map_kpts = mem.alloc<float>(static_cast<size_t>(K) * 2); map_kscores = mem.alloc<float>(K);
    map_D = mem.alloc<float>(static_cast<size_t>(K) * 256);
    q_kpts = mem.alloc<float>(static_cast<size_t>(B) * K * 2); q_kscores = mem.alloc<float>(static_cast<size_t>(B) * K);
    q_D = mem.alloc<float>(static_cast<size_t>(B) * K * 256);
    if (rc != MFR_OK) return rc;

    // ---- SuperPoint (superpoint.py:145-196) on the N frames of `im` -> counts, keypoints, scores, descriptors
    auto superpoint = [&](float* im, int N, int* counts_, float* kpts_, float* kscores_, float* D_) {
    {
      float *w = weights["conv1a.w"], *b = weights["conv1a.b"]; const int n = N, hh = H, ww = W;
      if (bf) push([=](cudaStream_t st) { return sp_conv1a_bf16(im, w, b, x1a, n, hh, ww, st); });
      else push([=](cudaStream_t st) { return sp_conv1a(im, w, b, x1a, n, hh, ww, st); });
    }
    auto pool = [&](float* in, float* out, int hh, int ww, int c) {
      const int n = N;
      if (bf) push([=](cudaStream_t st) { return maxpool2x2_bf16(in, out, n, hh, ww, c, st); });
      else push([=](cudaStream_t st) { return maxpool2x2(in, out, n, hh, ww, c, st); });
    };
    const int b16 = bf ? 1 : 0;   // bf16 operands (and outputs, up to the heads' inputs) in bf16 mode
    gemm("conv1b", x1a, N, H, W, 64, 64, 64, 3, ACT_RELU, nullptr, x1b, 64, 0, b16, b16);
    pool(x1b, p1, H, W, 64);
    gemm("conv2a", p1, N, H2, W2, 64, 64, 64, 3, ACT_RELU, nullptr, x2a, 64, 0, b16, b16);
    gemm("conv2b", x2a, N, H2, W2, 64, 64, 64, 3, ACT_RELU, nullptr, x2b, 64, 0, b16, b16);
    pool(x2b, p2, H2, W2, 64);
    gemm("conv3a", p2, N, H4, W4, 64, 64, 128, 3, ACT_RELU, nullptr, x3a, 128, 0, b16, b16);
    gemm("conv3b", x3a, N, H4, W4, 128, 128, 128, 3, ACT_RELU, nullptr, x3b, 128, 0, b16, b16);
    pool(x3b, p3, H4, W4, 128);
    gemm("conv4a", p3, N, h8, w8, 128, 128, 128, 3, ACT_RELU, nullptr, x4a, 128, 0, b16, b16);
    gemm("conv4b", x4a, N, h8, w8, 128, 128, 128, 3, ACT_RELU, nullptr, x4b, 128, 0, b16, b16);
    gemm("convPa", x4b, N, h8, w8, 128, 128, 256, 3, ACT_RELU, nullptr, cPa, 256, 0, b16, b16);
    gemm("convPb", cPa, N, h8, w8, 256, 256, 65, 1, ACT_NONE, nullptr, logits, 65, 0, b16, 0);
    {
      const int n = N, hh = h8, ww = w8, r = nms_r, bd = border, kk = K; const float th = kp_thr;
      float* kp = kpts_; float* ks = kscores_; int* cn = counts_;
      push([=](cudaStream_t st) { return sp_score_map(logits, 65, scores, n, hh, ww, st); });
      push([=](cudaStream_t st) { return sp_nms(scores, mask, t0, t1, t2, t3, n, hh * 8, ww * 8, r, st); }, 15);
      push([=](cudaStream_t st) { return sp_select_keypoints(scores, mask, n, hh * 8, ww * 8, th, bd, kk, kp, ks, cn, st); });
    }
    gemm("convDa", x4b, N, h8, w8, 128, 128, 256, 3, ACT_RELU, nullptr, cDa, 256, 0, b16, b16);
    gemm("convDb", cDa, N, h8, w8, 256, 256, 256, 1, ACT_NONE, nullptr, dense, 256, 0, b16, 0);
    {
      const int n = N, hh = h8, ww = w8, kk = K; float* kp = kpts_; int* cn = counts_; float* Dp = D_;
      const size_t rws = static_cast<size_t>(N) * h8 * w8;
      push([=](cudaStream_t st) { return l2norm256(dense, rws, st); });
      push([=](cudaStream_t st) { return sp_sample_descriptors(dense, kp, cn, n, hh, ww, kk, Dp, 256, st); });
    }
    };
    superpoint(img, NI, counts, kpts, kscores, D);
    // ---- SuperGlue (superglue.py:228-283). Token buffer X: [NI][K][512] = [desc | message]
    sg_begin = steps.size();
    {
      float* kp = kpts; float* ks = kscores; const int tot = NI * K, hh = H, ww = W;
      push([=](cudaStream_t st) { return sg_kenc_input(kp, ks, kin, tot, hh, ww, st); });
    }
    gemm("kenc.0", kin, NI, 1, K, 4, 4, 32, 1, ACT_RELU, nullptr, k1, 32);
    gemm("kenc.1", k1, NI, 1, K, 32, 32, 64, 1, ACT_RELU, nullptr, k2, 64);
    gemm("kenc.2", k2, NI, 1, K, 64, 64, 128, 1, ACT_RELU, nullptr, k3, 128);
    gemm("kenc.3", k3, NI, 1, K, 128, 128, 256, 1, ACT_RELU, nullptr, k4, 256);
    gemm("kenc.4", k4, NI, 1, K, 256, 256, 256, 1, ACT_NONE, D, X, 512, 256);   // X[:, :256] = desc + kenc
    if (bf) build_gnn_bf16(qkv, msg, h1, Xb);
    else for (int i = 0; i < 18; ++i) {   // tf32 / fp32x3 GNN layers
      const std::string p = "gnn." + std::to_string(i);
      gemm(p + ".qkv", X, NI, 1, K, 256, 512, 768, 1, ACT_NONE, nullptr, qkv, 768);
      {
        // multi-head softmax attention (superglue.py:85-89) as two tensor-core GEMMs with the heads as the H dimension:
        //   S[img][h][q][k] = Q_h K_h^T / 8   (B operand = keys of image img ^ cross, head h)
        //   P = softmax_k(S) in place, masked to the source image's keypoint count
        //   msg[img][q][64 h + d] = sum_k P[img][h][q][k] V[img ^ cross][k][64 h + d]   (B operand = V^T of that image / head)
        const int cross = i % 2, kk = K, n = NI; int* cn = counts;
        ConvGemmDesc d{};
        d.x = qkv; d.N = NI; d.H = 4; d.W = K; d.Cin = 64; d.ldx = 768; d.x_y_stride = 64; d.x_img_stride = static_cast<long long>(K) * 768;
        d.w = qkv + 256; d.Cout = K; d.R = 1; d.S = 1; d.stride = 1; d.pad = 0;
        d.b_batched = 2; d.ldw = 768; d.w_y_stride = 64; d.w_img_stride = static_cast<long long>(K) * 768; d.b_xor = cross;
        d.act = ACT_NONE; d.alpha = 0.125f; d.out = Sat; d.ldo = K; d.ldr = K;
        if (precision == 2) {   // q / k heads (64 channels each) -> [hi | lo | hi] / [hi | hi | lo] of 192, rows keep a stride of 768
          float *q3 = x3, *k3 = x3 + static_cast<size_t>(NI) * K * 768; const int rows = NI * K;
          if (rows > 65535) return MFR_ERR_ARG;
          push([=](cudaStream_t st) { return rows_split3(qkv, 64, 768, q3, 4, rows, 64, 0, nullptr, st); });
          push([=](cudaStream_t st) { return rows_split3(qkv + 256, 64, 768, k3, 4, rows, 64, 1, nullptr, st); });
          d.x = q3; d.Cin = 192; d.x_y_stride = 192;
          d.w = k3; d.w_y_stride = 192;
        }
        ConvGemmParams pq;
        int r = conv_gemm_build(d, &pq);
        if (r != MFR_OK) return r;
        push([pq](cudaStream_t st) { return conv_gemm_launch(pq, st); });
        push([=](cudaStream_t st) { return sg_softmax_rows(Sat, cn, cross, kk, n, st); });
        push([=](cudaStream_t st) { return sg_transpose_v(qkv, 768, Vt, kk, n, st); });
        ConvGemmDesc e{};
        e.x = Sat; e.N = NI; e.H = 4; e.W = K; e.Cin = K; e.ldx = K;
        e.w = Vt; e.Cout = 64; e.R = 1; e.S = 1; e.stride = 1; e.pad = 0;
        e.b_batched = 2; e.ldw = K; e.w_y_stride = 64LL * K; e.w_img_stride = 256LL * K; e.b_xor = cross;
        e.act = ACT_NONE; e.alpha = 1.f; e.out = msg; e.ldo = 256; e.ldr = 256; e.out_y_stride = 64;
        e.out_img_stride = static_cast<long long>(K) * 256;
        if (precision == 2) {   // P rows [K] -> [3K] (A pattern), V^T rows [K] -> [3K] (B pattern)
          float *p3 = x3, *v3 = x3 + static_cast<size_t>(NI) * 4 * K * 3 * K;
          const long long prow = static_cast<long long>(NI) * 4 * K, vrow = static_cast<long long>(NI) * 256;
          push([=](cudaStream_t st) { return rows_split3(Sat, kk, 0, p3, prow, 1, kk, 0, nullptr, st); });
          push([=](cudaStream_t st) { return rows_split3(Vt, kk, 0, v3, vrow, 1, kk, 1, nullptr, st); });
          e.x = p3; e.Cin = 3 * K; e.ldx = 3 * K;
          e.w = v3; e.ldw = 3 * K; e.w_y_stride = 64LL * 3 * K; e.w_img_stride = 256LL * 3 * K;
        }
        ConvGemmParams pv;
        r = conv_gemm_build(e, &pv);
        if (r != MFR_OK) return r;
        push([pv](cudaStream_t st) { return conv_gemm_launch(pv, st); });
      }
      gemm(p + ".merge", msg, NI, 1, K, 256, 256, 256, 1, ACT_NONE, nullptr, X + 256, 512);
      gemm(p + ".mlp0", X, NI, 1, K, 512, 512, 512, 1, ACT_RELU, nullptr, h1, 512);
      gemm(p + ".mlp3", h1, NI, 1, K, 512, 512, 256, 1, ACT_NONE, X, X, 512);   // x + delta (in place)
    }
    gemm("final_proj", X, NI, 1, K, 256, 512, 256, 1, ACT_NONE, nullptr, Mb, 256);
    {
      ConvGemmDesc d{};
      d.x = Mb; d.N = B; d.H = 1; d.W = K; d.Cin = 256; d.ldx = 256; d.x_img_stride = 2LL * K * 256;
      d.w = Mb + static_cast<size_t>(K) * 256; d.Cout = K; d.R = 1; d.S = 1; d.stride = 1; d.pad = 0;
      d.b_batched = 1; d.ldw = 256; d.w_img_stride = 2LL * K * 256; d.act = ACT_NONE; d.alpha = 1.f / 16.f;
      d.out = S; d.ldo = K; d.ldr = K;
      if (precision == 2) {   // matching descriptors of all images, once in the A pattern and once in the B pattern
        const long long rows = static_cast<long long>(NI) * K;
        float *ma = x3, *mb = x3 + static_cast<size_t>(rows) * 768;
        push([=](cudaStream_t st) { return rows_split3(Mb, 256, 0, ma, rows, 1, 256, 0, nullptr, st); });
        push([=](cudaStream_t st) { return rows_split3(Mb, 256, 0, mb, rows, 1, 256, 1, nullptr, st); });
        d.x = ma; d.Cin = 768; d.ldx = 768; d.x_img_stride = 2LL * K * 768;
        d.w = mb + static_cast<size_t>(K) * 768; d.ldw = 768; d.w_img_stride = 2LL * K * 768;
      }
      ConvGemmParams p;
      int r = conv_gemm_build(d, &p);
      if (r != MFR_OK) return r;
      push([p](cudaStream_t st) { return conv_gemm_launch(p, st); });
    }
    {
      const int kk = K, nb = B, iters = sk_iters; int* cn = counts; float* kp = kpts; const float th = match_thr;
      int* m0 = matches0; float* ms = mscores0; float *a0 = mk0, *a1 = mk1; int* mo = m_offsets;
      SpsgEngine* self = this;
      push([=](cudaStream_t st) { return sg_sinkhorn(S, kk, cn, self->bin_score, iters, kk, nb, u, v, st); }, 2 + 2 * sk_iters);
      push([=](cudaStream_t st) {
        return sg_extract_matches(S, kk, cn, u, v, th, kp, kk, rmax, rarg, carg, m0, ms, a0, a1, mo, nb, st);
      }, 3);
    }
    if (rc != MFR_OK) return rc;

    // ---- shared map frame
    LaunchList paired = std::move(steps);
    steps = LaunchList();
    superpoint(img, 1, map_counts, map_kpts, map_kscores, map_D);   // the map image is staged in frame 0
    map_steps = std::move(steps);
    steps = LaunchList();
    superpoint(img, B, q_counts, q_kpts, q_kscores, q_D);            // the queries in frames 0 .. B-1
    {
      int *mc = map_counts, *qc = q_counts, *cn = counts; const int nb = B, kk = K;
      float *mk = map_kpts, *ms = map_kscores, *md = map_D, *qk = q_kpts, *qs = q_kscores, *qd = q_D;
      float *kp = kpts, *ks = kscores, *Dp = D;
      push([=](cudaStream_t st) { return sp_pair_interleave(mc, mk, ms, md, qc, qk, qs, qd, nb, kk, cn, kp, ks, Dp, st); });
    }
    steps.append(paired, sg_begin, paired.steps.size());
    shared_steps = std::move(steps);
    steps = std::move(paired);
    return rc;
  }

  // the 18 GNN layers in bf16 mode. The fp32 token stream X [NI][K][512] keeps x in its first 256 columns; its bf16
  // shadow Xb [NI][K][512] = [x | message] is the operand of qkv and mlp.0. Per layer: qkv (bf16), the fused attention
  // (sg_attention.cu) into msg, merge into the message half of Xb, mlp.0 (ReLU) into h1, mlp.3 added to X in fp32, and
  // the x half of Xb refreshed from X (not after the last layer: final_proj reads X).
  void build_gnn_bf16(float* qkv, float* msg, float* h1, float* Xb) {
    const long long rows = static_cast<long long>(NI) * K;
    float* x = X;
    push([=](cudaStream_t st) { return rows_to_bf16(x, 512, Xb, 512, rows, 256, nullptr, st); });
    float* xb_msg = reinterpret_cast<float*>(reinterpret_cast<unsigned short*>(Xb) + 256);
    for (int i = 0; i < 18; ++i) {
      const std::string p = "gnn." + std::to_string(i);
      gemm(p + ".qkv", Xb, NI, 1, K, 256, 512, 768, 1, ACT_NONE, nullptr, qkv, 768, 0, 1, 1);
      SgAttentionParams ap;
      int r = sg_attention_build(qkv, 768, counts, NI, K, i % 2, msg, 256, &ap);
      if (r != MFR_OK) { rc = r; return; }
      push([ap](cudaStream_t st) { return sg_attention_launch(ap, st); });
      gemm(p + ".merge", msg, NI, 1, K, 256, 256, 256, 1, ACT_NONE, nullptr, xb_msg, 512, 0, 1, 1);
      gemm(p + ".mlp0", Xb, NI, 1, K, 512, 512, 512, 1, ACT_RELU, nullptr, h1, 512, 0, 1, 1);
      gemm(p + ".mlp3", h1, NI, 1, K, 512, 512, 256, 1, ACT_NONE, X, X, 512, 0, 1, 0);   // x + delta (fp32, in place)
      if (i < 17) push([=](cudaStream_t st) { return rows_to_bf16(x, 512, Xb, 512, rows, 256, nullptr, st); });
    }
  }

  // brings the derived weights and bin_score up to the last upload; runs outside any capture
  int prepare(cudaStream_t st) {
    if (bin_gen != weights.generation) {
      MFR_CUDA_CHECK(cudaMemcpy(&bin_score, weights["bin_score"], sizeof(float), cudaMemcpyDeviceToHost));
      bin_gen = weights.generation;
    }
    return derived.rebuild(weights, st);
  }

  // img0/img1: device [B][H][W]; copied into the pair-interleaved frame buffer
  int forward(const float* img0, const float* img1, cudaStream_t st) {
    if (!weights.complete()) return MFR_ERR_ARG;
    const size_t hw = static_cast<size_t>(H) * W;
    MFR_CUDA_CHECK(cudaMemcpy2DAsync(img, 2 * hw * 4, img0, hw * 4, hw * 4, B, cudaMemcpyDeviceToDevice, st));
    MFR_CUDA_CHECK(cudaMemcpy2DAsync(img + hw, 2 * hw * 4, img1, hw * 4, hw * 4, B, cudaMemcpyDeviceToDevice, st));
    const int r = prepare(st);
    if (r != MFR_OK) return r;
    return graph.launch(steps, st, use_graph, "spsg");
  }

  // Runs SuperPoint (eagerly) on one map image [H][W]; forward_shared reads its keypoints until the next set_map or
  // weight upload.
  int set_map(const float* img0, cudaStream_t st) {
    if (!weights.complete()) return MFR_ERR_ARG;
    map_gen = -1;
    MFR_CUDA_CHECK(cudaMemcpyAsync(img, img0, static_cast<size_t>(H) * W * 4, cudaMemcpyDeviceToDevice, st));
    int r = prepare(st);
    if (r == MFR_OK) r = map_steps.run(st);
    if (r != MFR_OK) return r;
    map_gen = weights.generation;
    return MFR_OK;
  }

  // forward(map repeated B times, img1) without running SuperPoint on the map again: the same bits in every output
  int forward_shared(const float* img1, cudaStream_t st) {
    if (!weights.complete() || map_gen != weights.generation) return MFR_ERR_ARG;
    MFR_CUDA_CHECK(cudaMemcpyAsync(img, img1, static_cast<size_t>(B) * H * W * 4, cudaMemcpyDeviceToDevice, st));
    const int r = prepare(st);
    if (r != MFR_OK) return r;
    return shared_graph.launch(shared_steps, st, use_graph, "spsg");
  }

  // SuperGlue only (the paired list from sg_begin on), on keypoints / scores / descriptors / counts uploaded by the
  // caller (host arrays, pair-interleaved image order) -- stage-boundary entry point for parity tests
  int forward_superglue(const int* h_counts, const float* h_kpts, const float* h_scores, const float* h_desc,
                        cudaStream_t st) {
    if (!weights.complete()) return MFR_ERR_ARG;
    MFR_CUDA_CHECK(cudaMemcpyAsync(counts, h_counts, sizeof(int) * NI, cudaMemcpyHostToDevice, st));
    MFR_CUDA_CHECK(cudaMemcpyAsync(kpts, h_kpts, sizeof(float) * NI * K * 2, cudaMemcpyHostToDevice, st));
    MFR_CUDA_CHECK(cudaMemcpyAsync(kscores, h_scores, sizeof(float) * NI * K, cudaMemcpyHostToDevice, st));
    MFR_CUDA_CHECK(cudaMemcpyAsync(D, h_desc, sizeof(float) * NI * K * 256, cudaMemcpyHostToDevice, st));
    const int r = prepare(st);
    if (r != MFR_OK) return r;
    return steps.run(st, sg_begin);
  }
};

int spsg_create(int B, int H, int W, int max_kp, int nms_radius, float kp_thr, int border, int sinkhorn_iters,
                float match_thr, int precision, SpsgEngine** out) {
  if (B < 1 || H < 64 || W < 64 || max_kp < 16 || max_kp > 2048 || (max_kp % 16)) return MFR_ERR_ARG;
  if (nms_radius < 0 || border < 0) return MFR_ERR_ARG;
  // 0 = TF32 GEMM inputs, 1 = bf16 operands and fused attention (see mfr_b200.h), 2 = 3xTF32 split (fp32-faithful)
  if (precision < 0 || precision > 2) return MFR_ERR_ARG;
  auto* e = new SpsgEngine();
  e->precision = precision;
  e->B = B; e->H = H; e->W = W; e->K = max_kp; e->nms_r = nms_radius; e->kp_thr = kp_thr; e->border = border;
  e->sk_iters = sinkhorn_iters; e->match_thr = match_thr;
  const int rc = e->build();
  if (rc != MFR_OK) { delete e; return rc; }
  *out = e;
  return MFR_OK;
}
void spsg_destroy(SpsgEngine* e) { delete e; }
EngineCore& engine_core(SpsgEngine* e) { return *e; }
int spsg_forward(SpsgEngine* e, const float* img0, const float* img1, cudaStream_t st) { return e->forward(img0, img1, st); }
int spsg_set_map(SpsgEngine* e, const float* img0, cudaStream_t st) { return e->set_map(img0, st); }
int spsg_forward_shared(SpsgEngine* e, const float* img1, cudaStream_t st) { return e->forward_shared(img1, st); }
void spsg_outputs(SpsgEngine* e, mfr_spsg_outputs* o) {
  o->counts = e->counts; o->keypoints = e->kpts; o->scores = e->kscores; o->descriptors = e->D; o->desc_ld = 256;
  o->matches0 = e->matches0; o->matching_scores0 = e->mscores0; o->m_offsets = e->m_offsets; o->mkpts0 = e->mk0;
  o->mkpts1 = e->mk1; o->max_keypoints = e->K;
}
int spsg_forward_superglue(SpsgEngine* e, const int* counts, const float* kpts, const float* scores, const float* desc,
                           cudaStream_t st) {
  return e->forward_superglue(counts, kpts, scores, desc, st);
}

}  // namespace mfr
