// LoFTR matcher engine: the whole coarse-to-fine network as a static launch list of hand-written
// sm_90a kernels (wgmma implicit-GEMM convs / linears + SIMT glue), replayed through a CUDA graph.
// Mirrors etc/feature_matching_baselines/LoFTR/src/loftr/loftr.py:29-75 of the reference
// (backbone -> pos-enc -> coarse transformer -> dual-softmax mutual-NN -> fine windows -> fine
// transformer -> expectation), for B image pairs per call, channel-last fp32 activations.
#include "loftr_engine.cuh"

#include <cstring>
#include <string>
#include <vector>

#include "conv_gemm.cuh"
#include "encoder_tail.cuh"
#include "engine_core.cuh"
#include "loftr_ops.cuh"

namespace mfr {

constexpr int kReservedLayers = 4;   // conv launches at the start of the list that leave LoftrEngine::reserved_sms SMs free

struct LoftrEngine : EngineCore {
  int B, H, W, NI;
  int H2, W2, H4, W4, H8, W8, L, Mcap;
  float thr, temperature;
  int border;
  int splits_kv = 96, splits_col = 32;   // splits_kv is set from the image count in build()
  int precision = 0;   // MFR_PRECISION_* (include/mfr_b200.h)
  // The pose back end of the previous batch runs on its own stream under the first layers of this batch's matcher. Its blocks
  // do not fit next to the persistent GEMM CTAs, and a persistent kernel with a static tile assignment whose CTA has to wait
  // for an SM is late by that CTA's whole share: the first kReservedLayers conv launches therefore leave `reserved_sms` SMs
  // free (0 = use every SM).
  int reserved_sms = 0;
  int conv_count = 0;
  DerivedWeights derived{&rc};   // precision 1: bf16 GEMM weights; precision 2: their [hi | hi | lo] split
  float* x3 = nullptr;         // precision 2: scratch for the [hi | lo | hi] split of a GEMM's activations
  size_t x3_cap = 0;
  int last_src_h = -1, last_src_w = -1;

  // `steps` is the paired forward; conv() and push() append to it.
  // Shared map frame (set_map / forward_shared): map_steps encodes one image up to coarse layer 0 into the map_*
  // buffers; shared_steps runs the query half of a batch, broadcasts the map into the image-0 half and continues with
  // the paired list's own steps from coarse layer 1 on.
  LaunchList map_steps, shared_steps;
  GraphExec graph, shared_graph;
  void push(const std::string& name, std::function<int(cudaStream_t)> f, int launches = 1) {
    steps.push(std::move(f), name, launches);
  }
  // buffers
  float* img = nullptr;
  float *a0, *a1, *a2, *b0, *b1, *b2, *c0, *c1, *c2, *fc, *p4a, *p4b, *p4c, *p2a, *p2b;
  float *tok, *qkv, *msg, *kvp, *kv, *S;
  float *mrg = nullptr, *h1 = nullptr, *h2 = nullptr;   // tf32 / fp32x3 only (unfused encoder tail)
  float *tokb = nullptr, *ftokb = nullptr;   // bf16 mode: bf16 shadows of tok / ftok (same shape; float-typed like the other bf16 buffers)
  size_t ftok_elems = 0;
  float *featf = nullptr;
  // the encoded map frame: its [H][W] input, tokens after coarse layer 0 ([L][512], + bf16 shadow), fine map [H/2][W/2][128]
  float *map_img = nullptr, *map_tok = nullptr, *map_tokb = nullptr, *map_featf = nullptr;
  long long map_gen = -1;   // weight generation the map was encoded with (-1: no map)
  int map_src_h = -1, map_src_w = -1;
  float* shadow(float* x) const {            // same element offset inside the shadow buffer
    if (x >= ftok && x < ftok + ftok_elems) return ftokb + (x - ftok) / 2;
    if (x >= map_tok && x < map_tok + static_cast<size_t>(L) * 512) return map_tokb + (x - map_tok) / 2;
    return tokb + (x - tok) / 2;
  }
  CoarseMatchBuffers cm;
  float *cin, *cproj, *win, *ftok, *fqkv, *fmsg, *mk1f, *expec;
  float *fmrg = nullptr, *fh1 = nullptr, *fh2 = nullptr;   // tf32 / fp32x3 only

  // ---- step builders -----------------------------------------------------------------------
  void conv(const std::string& wname, const float* x, int N, int Hh, int Ww, int Cin, long long ldx,
            int Cout, int R, int stride, bool bias, const float* residual, int act, float* out,
            long long ldo, int act_cols = 0, const int* dyn_w = nullptr, const float* w_override = nullptr,
            const float* bias_override = nullptr, int in_bf16 = 0, int out_bf16 = 0, int w_rows_total = 0,
            int w_row_off = 0) {
    ConvGemmDesc d{};
    int cin_gemm = Cin;                       // K of the GEMM per tap (3 * Cin in the 3xTF32 mode)
    // a GEMM may use a row window [w_row_off, w_row_off + Cout) of a larger weight (q / k|v parts of qkv); cross layers
    // ask for the same weights twice and share one derived copy
    const long long w_rows = static_cast<long long>(w_rows_total > 0 ? w_rows_total : Cout) * R * R;
    if (precision == 2 && !in_bf16) {
      // fp32-faithful mode: A = [hi | lo | hi] of the activations (split into the scratch x3 right before the GEMM),
      // B = [hi | hi | lo] of the weights (derived, rebuilt after every weight upload) -> one TF32 GEMM over 3 * Cin
      const long long rows_img = static_cast<long long>(Hh) * Ww;
      if (static_cast<size_t>(N) * rows_img * 3 * Cin > x3_cap) {
        fprintf(stderr, "[mfr_b200] split scratch too small for %s\n", wname.c_str());
        rc = MFR_ERR_ARG;
        return;
      }
      float* x3_ = x3; const float* xs = x; const int N_ = N, C_ = Cin; const long long ldx_ = ldx;
      push("split3", [=](cudaStream_t st) { return rows_split3(xs, ldx_, rows_img * ldx_, x3_, rows_img, N_, C_, 0, dyn_w, st); });
      w_override = derived.get(weights, wname + ".w", w_rows, Cin, static_cast<long long>(w_row_off) * R * R);
      x = x3; ldx = 3 * Cin; cin_gemm = 3 * Cin;
    }
    d.x = x; d.N = N; d.H = Hh; d.W = Ww; d.Cin = cin_gemm; d.ldx = ldx;
    d.in_bf16 = in_bf16; d.out_bf16 = out_bf16;
    if (in_bf16) {   // bf16 copy of the weights, Cin padded to a multiple of 8 (16-byte TMA strides)
      d.ldw = derived.ld(Cin);
      w_override = derived.get(weights, wname + ".w", w_rows, Cin, static_cast<long long>(w_row_off) * R * R);
    }
    d.w = w_override ? w_override : weights[wname + ".w"];
    d.Cout = Cout; d.R = R; d.S = R; d.stride = stride; d.pad = R / 2;
    d.b_batched = 0; if (!in_bf16) d.ldw = 0; d.act_cols = act_cols; d.dyn_w = dyn_w;
    d.bias = bias ? (bias_override ? bias_override : weights[wname + ".b"]) : nullptr;
    d.residual = residual; d.ldr = ldo;
    d.act = act; d.alpha = 1.f; d.out = out; d.ldo = ldo;
    ConvGemmParams p;
    const int r = conv_gemm_build(d, &p);
    if (r != MFR_OK) { rc = r; return; }
    if (reserved_sms > 0 && conv_count < kReservedLayers) p.grid_limit = conv_gemm_num_sms() - reserved_sms;
    ++conv_count;
    Step& s = steps.push([p](cudaStream_t st) { return conv_gemm_launch(p, st); }, wname.empty() ? "qkv" : wname);
    s.kind = 1;
    s.dyn_rows = dyn_w;
    s.dyn_images = N;
    const double per_pixel = 2.0 * Cout * Cin * R * R;
    s.flops = dyn_w ? per_pixel : per_pixel * N * p.Ho * p.Wo;
  }

  void specs_backbone() {
    weights.add("stem.w", 128 * 49);
    weights.add("stem.b", 128);
    auto cv = [&](const std::string& n, int cin, int cout, int r, bool bias) {
      weights.add(n + ".w", static_cast<size_t>(cout) * r * r * cin);
      if (bias) weights.add(n + ".b", cout);
    };
    int cin = 128;
    const int dims[3] = {128, 196, 256};
    for (int li = 0; li < 3; ++li) {
      const int c = dims[li];
      for (int bi = 0; bi < 2; ++bi) {
        const std::string p = "layer" + std::to_string(li + 1) + "." + std::to_string(bi);
        cv(p + ".conv1", bi == 0 ? cin : c, c, 3, true);
        cv(p + ".conv2", c, c, 3, true);
        if (bi == 0 && li > 0) cv(p + ".down", cin, c, 1, true);
      }
      cin = c;
    }
    cv("layer3_outconv", 256, 256, 1, false);
    cv("layer2_outconv", 196, 256, 1, false);
    cv("layer2_outconv2.0", 256, 256, 3, true);
    cv("layer2_outconv2.3", 256, 196, 3, false);
    cv("layer1_outconv", 128, 196, 1, false);
    cv("layer1_outconv2.0", 196, 196, 3, true);
    cv("layer1_outconv2.3", 196, 128, 3, false);
    weights.add("pos_enc", static_cast<size_t>(L) * 256);
  }
  void specs_transformer(const std::string& pre, int C, int layers) {
    for (int i = 0; i < layers; ++i) {
      const std::string p = pre + "." + std::to_string(i);
      weights.add(p + ".qkv.w", static_cast<size_t>(3) * C * C);
      weights.add(p + ".merge.w", static_cast<size_t>(C) * C);
      weights.add(p + ".mlp0.w", static_cast<size_t>(4) * C * C);
      weights.add(p + ".mlp2.w", static_cast<size_t>(2) * C * C);
      weights.add(p + ".norm1.g", C);
      weights.add(p + ".norm1.b", C);
      weights.add(p + ".norm2.g", C);
      weights.add(p + ".norm2.b", C);
    }
  }

  // One LoFTREncoderLayer (transformer.py:35-58) on `n` "images" of `rows` tokens each.
  //   x, src : token buffers with row stride 2C (cols [0,C) = features, [C,2C) = message scratch)
  //   q/k/v live in `qkv_x` / `qkv_s` (row stride 3C) at the rows of the x / src images.
  //   mrg_x, h1_x, h2_x : scratch of the unfused tail (tf32 / fp32x3 only, null in bf16 mode)
  void encoder_layer(const std::string& p, int C, float* x, float* src, float* qkv_x, float* qkv_s,
                     float* msg_x, float* mrg_x, float* h1_x, float* h2_x, int n, int rows,
                     const int* dyn_rows, const int* dyn_items, bool windows, int kv_splits = 0) {
    float* wq = weights[p + ".qkv.w"];
    const long long ld2 = 2 * C, ld3 = 3 * C;
    // bf16 mode: q|k|v and the attention message are stored in bf16 — these GEMMs and the attention kernels are
    // HBM-bound — while the residual stream, LayerNorm inputs and outputs stay fp32.
    // The buffers are float-typed: `tb` bf16 elements per float when converting element offsets.
    const int tbf = precision == 1 ? 1 : 0, tb = tbf ? 2 : 1;
    auto E = [tb](float* ptr, size_t elems) { return ptr + elems / tb; };
    // bf16 mode: the q|k|v GEMMs take their A operand from the bf16 shadow of the token stream (written by the fused
    // tail): half the operand bytes and kind::f16 MMAs instead of kind::tf32. They store the raw projections, and the
    // attention kernels apply elu + 1 to their mma fragments.
    float* xb = tbf ? shadow(x) : x;
    float* srcb = tbf ? shadow(src) : src;
    const std::string qn = p + ".qkv";
    const int qk_act = tbf ? ACT_NONE : ACT_ELU1;
    if (x == src) {
      conv(qn, xb, n, 1, rows, C, ld2, 3 * C, 1, 1, false, nullptr, qk_act, qkv_x, ld3, 2 * C, dyn_rows, wq, nullptr, tbf, tbf,
           3 * C, 0);
    } else {
      conv(qn, xb, n, 1, rows, C, ld2, C, 1, 1, false, nullptr, qk_act, qkv_x, ld3, C, dyn_rows, wq, nullptr, tbf, tbf, 3 * C, 0);
      conv(qn, srcb, n, 1, rows, C, ld2, 2 * C, 1, 1, false, nullptr, qk_act, E(qkv_s, C), ld3, C, dyn_rows,
           wq + static_cast<size_t>(C) * C, nullptr, tbf, tbf, 3 * C, C);
    }
    if (!windows) {
      float* kvp_ = kvp; float* kv_ = kv;
      // same partial-buffer footprint for n = B or n = 2B images, unless the caller pins the split count
      const int Lr = rows, sk = kv_splits > 0 ? kv_splits : splits_kv * NI / n;
      float *kp = E(qkv_s, C), *vp = E(qkv_s, 2 * C);
      push("attn_long", [=](cudaStream_t st) {
        return linear_attention_long(qkv_x, ld3, kp, ld3, vp, ld3, msg_x, C, kvp_, kv_, n, Lr, Lr, 8, 32, sk, st, tbf);
      }, 3);
    } else {
      const int items_cap = rows / 25;
      for (int side = 0; side < n; ++side) {
        const size_t off3 = static_cast<size_t>(side) * rows * ld3;
        const size_t off1 = static_cast<size_t>(side) * rows * C;
        float *qp = E(qkv_x, off3), *kp = E(qkv_s, off3 + C), *vp = E(qkv_s, off3 + 2 * C), *mp = E(msg_x, off1);
        push("attn_windows", [=](cudaStream_t st) {
          return linear_attention_windows(qp, ld3, kp, ld3, vp, ld3, mp, C, dyn_items, items_cap, 25, st, tbf);
        });
      }
    }
    const float *g1 = weights[p + ".norm1.g"], *b1 = weights[p + ".norm1.b"];
    const float *g2 = weights[p + ".norm2.g"], *b2 = weights[p + ".norm2.b"];
    if (tbf) {
      // merge -> norm1 -> mlp([x | message]) -> norm2 -> residual as ONE kernel: the merge output, the norm1 output, the
      // 2C-wide hidden tensor and the mlp output never leave the SM (encoder_tail.cu)
      EncoderTailDesc d{};
      d.msg = msg_x; d.ld_msg = C; d.xb_in = xb; d.ld_xb = ld2;
      d.w_merge = derived.get(weights, p + ".merge.w", C, C);
      d.w_mlp0 = derived.get(weights, p + ".mlp0.w", 2 * C, 2 * C);
      d.w_mlp2 = derived.get(weights, p + ".mlp2.w", C, 2 * C);
      d.g1 = g1; d.b1 = b1; d.g2 = g2; d.b2 = b2; d.x = x; d.ldx = ld2; d.C = C;
      if (dyn_rows) { d.n_img = n; d.rows_cap = rows; d.dyn_rows = dyn_rows; }
      else { d.n_img = 1; d.rows_cap = static_cast<long long>(n) * rows; d.dyn_rows = nullptr; }
      EncoderTailParams tp;
      const int r = encoder_tail_build(d, &tp);
      if (r != MFR_OK) { rc = r; return; }
      Step& s = steps.push([tp](cudaStream_t st) { return encoder_tail_launch(tp, st); }, p + ".tail");
      s.kind = 1;
      s.dyn_rows = dyn_rows;
      s.dyn_images = n;
      const double per_row = 14.0 * C * C;      // 2 * (C*C + 2C*2C + 2C*C)
      s.flops = dyn_rows ? per_row : per_row * n * rows;
      return;
    }
    // tf32 / fp32x3: merge, norm1 into the message half of x, mlp0 on [x | message], mlp2, norm2 + residual
    conv(p + ".merge", msg_x, n, 1, rows, C, C, C, 1, 1, false, nullptr, ACT_NONE, mrg_x, C, 0, dyn_rows);
    const long long tot = static_cast<long long>(n) * rows;
    if (dyn_rows == nullptr) {
      push("layernorm", [=](cudaStream_t st) {
        return layernorm_rows(mrg_x, C, g1, b1, nullptr, 0, x + C, ld2, tot, C, nullptr, st);
      });
    } else {
      for (int side = 0; side < n; ++side) {
        const size_t o1 = static_cast<size_t>(side) * rows * C, o2 = static_cast<size_t>(side) * rows * ld2;
        push("layernorm", [=](cudaStream_t st) {
          return layernorm_rows(mrg_x + o1, C, g1, b1, nullptr, 0, x + o2 + C, ld2, rows, C, dyn_rows, st);
        });
      }
    }
    conv(p + ".mlp0", x, n, 1, rows, 2 * C, ld2, 2 * C, 1, 1, false, nullptr, ACT_RELU, h1_x, ld2, 0, dyn_rows);
    conv(p + ".mlp2", h1_x, n, 1, rows, 2 * C, ld2, C, 1, 1, false, nullptr, ACT_NONE, h2_x, C, 0, dyn_rows);
    if (dyn_rows == nullptr) {
      push("layernorm", [=](cudaStream_t st) {
        return layernorm_rows(h2_x, C, g2, b2, x, ld2, x, ld2, tot, C, nullptr, st);
      });
    } else {
      for (int side = 0; side < n; ++side) {
        const size_t o1 = static_cast<size_t>(side) * rows * C, o2 = static_cast<size_t>(side) * rows * ld2;
        push("layernorm", [=](cudaStream_t st) {
          return layernorm_rows(h2_x + o1, C, g2, b2, x + o2, ld2, x + o2, ld2, rows, C, dyn_rows, st);
        });
      }
    }
  }

  // Stem + ResNet-FPN (resnet_fpn.py:100-119) over the N images of `input` ([N][H][W]): the 1/8 map goes to feat_c
  // ([N][L][256] fp32), the 1/2 map to feat_f ([N][H/2][W/2][128] fp32). The other activations live in the shared
  // scratch buffers a0 ... p2b.
  void backbone(float* input, int N, float* feat_c, float* feat_f) {
    const bool bf = precision == 1;
    const int c196 = bf ? 200 : 196;
    const int B16 = bf ? 1 : 0;
    {
      float *img_ = input, *a0_ = a0; float* ws = weights["stem.w"]; float* bs = weights["stem.b"];
      const int NI_ = N, H_ = H, W_w = W, ob = B16, exact = precision == 2 ? 1 : 0;
      push("stem", [=](cudaStream_t st) { return stem_conv7x7(img_, ws, bs, a0_, NI_, H_, W_w, st, ob, exact); });
    }
    auto bconv = [&](const std::string& name, const float* x, int Hh, int Ww, int Cin, int ldx, int Cout, int R,
                     int stride, bool bias, const float* res, int act, float* out, int ldo, int out16) {
      conv(name, x, N, Hh, Ww, Cin, ldx, Cout, R, stride, bias, res, act, out, ldo, 0, nullptr, nullptr, nullptr, B16,
           out16);
    };
    bconv("layer1.0.conv1", a0, H2, W2, 128, 128, 128, 3, 1, true, nullptr, ACT_RELU, a1, 128, B16);
    bconv("layer1.0.conv2", a1, H2, W2, 128, 128, 128, 3, 1, true, a0, ACT_RELU, a2, 128, B16);
    bconv("layer1.1.conv1", a2, H2, W2, 128, 128, 128, 3, 1, true, nullptr, ACT_RELU, a1, 128, B16);
    bconv("layer1.1.conv2", a1, H2, W2, 128, 128, 128, 3, 1, true, a2, ACT_RELU, a0, 128, B16);  // x1 = a0
    bconv("layer2.0.conv1", a0, H2, W2, 128, 128, 196, 3, 2, true, nullptr, ACT_RELU, b1, c196, B16);
    bconv("layer2.0.down", a0, H2, W2, 128, 128, 196, 1, 2, true, nullptr, ACT_NONE, b2, c196, B16);
    bconv("layer2.0.conv2", b1, H4, W4, 196, c196, 196, 3, 1, true, b2, ACT_RELU, b0, c196, B16);
    bconv("layer2.1.conv1", b0, H4, W4, 196, c196, 196, 3, 1, true, nullptr, ACT_RELU, b1, c196, B16);
    bconv("layer2.1.conv2", b1, H4, W4, 196, c196, 196, 3, 1, true, b0, ACT_RELU, b2, c196, B16);  // x2 = b2
    bconv("layer3.0.conv1", b2, H4, W4, 196, c196, 256, 3, 2, true, nullptr, ACT_RELU, c1, 256, B16);
    bconv("layer3.0.down", b2, H4, W4, 196, c196, 256, 1, 2, true, nullptr, ACT_NONE, c2, 256, B16);
    bconv("layer3.0.conv2", c1, H8, W8, 256, 256, 256, 3, 1, true, c2, ACT_RELU, c0, 256, B16);
    bconv("layer3.1.conv1", c0, H8, W8, 256, 256, 256, 3, 1, true, nullptr, ACT_RELU, c1, 256, B16);
    bconv("layer3.1.conv2", c1, H8, W8, 256, 256, 256, 3, 1, true, c0, ACT_RELU, c2, 256, B16);  // x3 = c2
    bconv("layer3_outconv", c2, H8, W8, 256, 256, 256, 1, 1, false, nullptr, ACT_NONE, feat_c, 256, 0);   // fp32 out
    bconv("layer2_outconv", b2, H4, W4, 196, c196, 256, 1, 1, false, nullptr, ACT_NONE, p4a, 256, B16);
    {
      float *s_ = feat_c, *d_ = p4a; const int n = N, hs = H8, wsz = W8, ob = B16;
      push("upsample", [=](cudaStream_t st) { return upsample2x_add(s_, d_, n, hs, wsz, 256, 256, 256, 0, ob, st); });
    }
    bconv("layer2_outconv2.0", p4a, H4, W4, 256, 256, 256, 3, 1, true, nullptr, ACT_LEAKY, p4b, 256, B16);
    bconv("layer2_outconv2.3", p4b, H4, W4, 256, 256, 196, 3, 1, false, nullptr, ACT_NONE, p4c, c196, B16);
    bconv("layer1_outconv", a0, H2, W2, 128, 128, 196, 1, 1, false, nullptr, ACT_NONE, p2a, c196, B16);
    {
      float *s_ = p4c, *d_ = p2a; const int n = N, hs = H4, wsz = W4, ld = c196, ob = B16;
      push("upsample", [=](cudaStream_t st) { return upsample2x_add(s_, d_, n, hs, wsz, 196, ld, ld, ob, ob, st); });
    }
    bconv("layer1_outconv2.0", p2a, H2, W2, 196, c196, 196, 3, 1, true, nullptr, ACT_LEAKY, p2b, c196, B16);
    bconv("layer1_outconv2.3", p2b, H2, W2, 196, c196, 128, 3, 1, false, nullptr, ACT_NONE, feat_f, 128, 0);   // fp32 out
  }

  // pos-enc add (loftr.py:58-59) of N images' 1/8 maps into token rows t (row stride 512), and its bf16 shadow
  void coarse_tokens(float* feat_c, int N, float* t) {
    float* pe = weights["pos_enc"]; const int n = N, l = L;
    push("posenc", [=](cudaStream_t st) { return posenc_tokens(feat_c, pe, t, 512, n, l, 256, st); });
    if (precision == 1) {
      float* tb_ = shadow(t);
      push("to_bf16", [=](cudaStream_t st) { return rows_to_bf16(t, 512, tb_, 512, static_cast<long long>(n) * l, 256, nullptr, st); });
    }
  }

  // Coarse layer 0 (a self layer) on n images of token rows t. The K'ᵀV sums are split into splits_kv parts whatever n
  // is — the split count of the paired list's self layers — so an image gives the same bits alone as inside a batch.
  void coarse_layer0(float* t, int n) {
    encoder_layer("coarse.0", 256, t, t, qkv, qkv, msg, mrg, h1, h2, n, L, nullptr, nullptr, false, splits_kv);
  }

  // 5x5 windows of the fine maps around every coarse match: side s reads pair b's map at feat_f_s + b * stride_s
  void fine_windows(const float* f0, long long stride0, const float* f1, long long stride1) {
    CoarseMatchBuffers cmb = cm; float *cproj_ = cproj, *win_ = win;
    const int Mc = Mcap, Hf = H2, Wf = W2, wc = W8;
    push("fine_gather_windows", [=](cudaStream_t st) {
      return fine_gather_windows(f0, stride0, f1, stride1, Hf, Wf, wc, cmb.b_ids, cmb.i_ids, cmb.j_ids, cmb.m_total, Mc,
                                 cproj_, win_, st);
    });
  }

  int build() {
    NI = 2 * B;
    H2 = H / 2; W2 = W / 2; H4 = H / 4; W4 = W / 4; H8 = H / 8; W8 = W / 8;
    L = H8 * W8;
    Mcap = B * L;
    specs_backbone();
    specs_transformer("coarse", 256, 8);
    weights.add("fine.down_proj.w", 128 * 256);
    weights.add("fine.down_proj.b", 128);
    weights.add("fine.merge_feat.w", 128 * 256);
    weights.add("fine.merge_feat.b", 128);
    specs_transformer("fine", 128, 2);
    weights.alloc(mem);

    const size_t px2 = static_cast<size_t>(NI) * H2 * W2, px4 = static_cast<size_t>(NI) * H4 * W4,
                 px8 = static_cast<size_t>(NI) * H8 * W8;
    img = mem.alloc<float>(static_cast<size_t>(NI) * H * W, "img");
    const bool bf = precision == 1;
    const int c196 = bf ? 200 : 196;                  // pixel stride of the 196-channel maps (16-byte rows in bf16)
    const size_t esz = bf ? 2 : 4;
    auto balloc = [&](size_t elems, const char* name) {  // backbone activation buffer (fp32 or bf16 storage)
      return reinterpret_cast<float*>(mem.alloc<unsigned char>(elems * esz, name));
    };
    if (bf) derived.alloc(mem, weights, DerivedWeights::kBf16);
    if (precision == 2) {
      derived.alloc(mem, weights, DerivedWeights::kSplit3);
      const size_t frows_ = static_cast<size_t>(2) * Mcap * 25;
      x3_cap = 3 * std::max(std::max(px2 * 196, px4 * 256), std::max(px8 * 512, frows_ * 256));
      x3 = mem.alloc<float>(x3_cap, "split3_scratch");
    }
    a0 = balloc(px2 * 128, "a0"); a1 = balloc(px2 * 128, "a1"); a2 = balloc(px2 * 128, "a2");
    b0 = balloc(px4 * c196, "b0"); b1 = balloc(px4 * c196, "b1"); b2 = balloc(px4 * c196, "b2");
    c0 = balloc(px8 * 256, "c0"); c1 = balloc(px8 * 256, "c1"); c2 = balloc(px8 * 256, "c2");
    fc = mem.alloc<float>(px8 * 256, "feat_c_backbone");
    p4a = balloc(px4 * 256, "p4a"); p4b = balloc(px4 * 256, "p4b"); p4c = balloc(px4 * c196, "p4c");
    p2a = balloc(px2 * c196, "p2a"); p2b = balloc(px2 * c196, "p2b");
    featf = mem.alloc<float>(px2 * 128, "feat_f");
    tok = mem.alloc<float>(px8 * 512, "tok");
    if (bf) tokb = reinterpret_cast<float*>(mem.alloc<unsigned short>(px8 * 512, "tok_bf16"));
    map_img = mem.alloc<float>(static_cast<size_t>(H) * W, "map_img");
    map_tok = mem.alloc<float>(static_cast<size_t>(L) * 512, "map_tok");
    if (bf) map_tokb = reinterpret_cast<float*>(mem.alloc<unsigned short>(static_cast<size_t>(L) * 512, "map_tok_bf16"));
    map_featf = mem.alloc<float>(static_cast<size_t>(H2) * W2 * 128, "map_feat_f");
    qkv = mem.alloc<float>(px8 * 768, "qkv"); msg = mem.alloc<float>(px8 * 256, "msg");
    if (!bf) {   // the unfused encoder tail's scratch (bf16 mode runs the fused tail)
      mrg = mem.alloc<float>(px8 * 256, "mrg"); h1 = mem.alloc<float>(px8 * 512, "h1"); h2 = mem.alloc<float>(px8 * 256, "h2");
    }
    splits_kv = std::max(1, std::min(L / 16, (2 * sm_count() + NI - 1) / NI));   // ~2 blocks per SM when all images run
    kvp = mem.alloc<float>(static_cast<size_t>(NI) * 8 * splits_kv * 1056, "kvp");
    kv = mem.alloc<float>(static_cast<size_t>(NI) * 8 * 1056, "kv");
    S = mem.alloc<float>(static_cast<size_t>(B) * L * L, "sim");
    const size_t BL = static_cast<size_t>(B) * L;
    cm.row_max = mem.alloc<float>(BL); cm.row_rsum = mem.alloc<float>(BL);
    cm.col_max = mem.alloc<float>(BL); cm.col_rsum = mem.alloc<float>(BL);
    splits_col = coarse_match_splits(B, L);
    cm.col_part = mem.alloc<float>(BL * splits_col * 2);
    cm.rconf_max = mem.alloc<float>(BL); cm.rconf_arg = mem.alloc<int>(BL); cm.rconf_ties = mem.alloc<int>(BL);
    cm.cconf_max = mem.alloc<float>(BL); cm.jsel = mem.alloc<int>(BL);
    cm.m_total = mem.alloc<int>(4); cm.m_offsets = mem.alloc<int>(B + 1);
    cm.b_ids = mem.alloc<int>(BL); cm.i_ids = mem.alloc<int>(BL); cm.j_ids = mem.alloc<int>(BL);
    cm.mconf = mem.alloc<float>(BL, "mconf"); cm.mkpts0_c = mem.alloc<float>(BL * 2, "mkpts0_c");
    cm.mkpts1_c = mem.alloc<float>(BL * 2, "mkpts1_c");
    const size_t frows = static_cast<size_t>(2) * Mcap * 25;
    cin = mem.alloc<float>(static_cast<size_t>(2) * Mcap * 256, "fine_cin");
    cproj = mem.alloc<float>(static_cast<size_t>(2) * Mcap * 128, "fine_cproj");
    win = mem.alloc<float>(frows * 256, "fine_win");
    ftok = mem.alloc<float>(frows * 256, "fine_tok");
    ftok_elems = frows * 256;
    if (bf) ftokb = reinterpret_cast<float*>(mem.alloc<unsigned short>(frows * 256, "fine_tok_bf16"));
    fqkv = mem.alloc<float>(frows * 384, "fine_qkv"); fmsg = mem.alloc<float>(frows * 128);
    if (!bf) { fmrg = mem.alloc<float>(frows * 128); fh1 = mem.alloc<float>(frows * 256); fh2 = mem.alloc<float>(frows * 128); }
    mk1f = mem.alloc<float>(BL * 2, "mkpts1_f"); expec = mem.alloc<float>(BL * 3, "expec_f");
    if (rc != MFR_OK) return rc;

    // ---------------------------------------------------------------- backbone, pos-enc, coarse layer 0
    conv_count = 0;
    backbone(img, NI, fc, featf);
    coarse_tokens(fc, NI, tok);
    coarse_layer0(tok, NI);
    const size_t img_f = static_cast<size_t>(H2) * W2 * 128;   // floats of one image's fine map
    const size_t half_tok = static_cast<size_t>(B) * L * 512, half_qkv = static_cast<size_t>(B) * L * 768;
    const size_t half_c = static_cast<size_t>(B) * L * 256, half_2c = static_cast<size_t>(B) * L * 512;
    const int tb = bf ? 2 : 1;   // qkv / msg hold bf16 in that mode (see encoder_layer)
    auto at = [](float* p, size_t off) { return p ? p + off : p; };   // the unfused tail's scratch is null in bf16 mode
    const size_t layer1_begin = steps.size();
    for (int i = 1; i < 8; ++i) {
      const std::string p = "coarse." + std::to_string(i);
      if (i % 2 == 0) {  // self: both image sets at once
        encoder_layer(p, 256, tok, tok, qkv, qkv, msg, mrg, h1, h2, NI, L, nullptr, nullptr, false);
      } else {  // cross: feat0 <- (feat0, feat1), then feat1 <- (feat1, updated feat0)
        encoder_layer(p, 256, tok, tok + half_tok, qkv, qkv + half_qkv / tb, msg, mrg, h1, h2, B, L, nullptr,
                      nullptr, false);
        encoder_layer(p, 256, tok + half_tok, tok, qkv + half_qkv / tb, qkv, msg + half_c / tb, at(mrg, half_c),
                      at(h1, half_2c), at(h2, half_c), B, L, nullptr, nullptr, false);
      }
    }

    // ---------------------------------------------------------------- coarse matching
    {
      ConvGemmDesc d{};
      d.x = tok; d.N = B; d.H = 1; d.W = L; d.Cin = 256; d.ldx = 512;
      d.w = tok + half_tok; d.Cout = L; d.R = 1; d.S = 1; d.stride = 1; d.pad = 0;
      // bf16 mode: the correlation reads the bf16 shadow of the final tokens (kind::f16, half the operand bytes)
      if (bf) { d.x = tokb; d.w = tokb + half_tok / 2; d.in_bf16 = 1; }
      if (precision == 2) {   // 3xTF32: X -> [hi | lo | hi], Y -> [hi | hi | lo], one GEMM over K = 768
        const size_t BLr = static_cast<size_t>(B) * L;
        float *xa = x3, *xb = x3 + BLr * 768; const float *t0 = tok, *t1 = tok + half_tok; const int B_ = B, L_ = L;
        push("split3", [=](cudaStream_t st) { return rows_split3(t0, 512, static_cast<long long>(L_) * 512, xa, L_, B_, 256, 0, nullptr, st); });
        push("split3", [=](cudaStream_t st) { return rows_split3(t1, 512, static_cast<long long>(L_) * 512, xb, L_, B_, 256, 1, nullptr, st); });
        d.x = xa; d.w = xb; d.Cin = 768; d.ldx = 768; d.ldw = 768;
      }
      d.b_batched = 1; if (precision != 2) d.ldw = 512; d.act = ACT_NONE; d.alpha = 1.f / (256.f * temperature);
      d.out = S; d.ldo = L; d.ldr = L;
      ConvGemmParams p;
      const int r = conv_gemm_build(d, &p);
      if (r != MFR_OK) return r;
      Step& s = steps.push([p](cudaStream_t st) { return conv_gemm_launch(p, st); }, "correlation");
      s.kind = 1;
      s.flops = 2.0 * B * static_cast<double>(L) * L * 256;
      CoarseMatchBuffers cmb = cm; float* S_ = S;
      const int B_ = B, L_ = L, hc = H8, wc = W8, bd = border, sc = splits_col; const float th = thr;
      const float scale = static_cast<float>(H) / static_cast<float>(H8);
      push("coarse_match", [=](cudaStream_t st) {
        return coarse_match(S_, cmb, B_, L_, hc, wc, th, bd, scale, sc, st);
      }, 8);
    }

    // ---------------------------------------------------------------- fine level
    {
      CoarseMatchBuffers cmb = cm; float *tok_ = tok, *cin_ = cin;
      const int B_ = B, L_ = L, Mc = Mcap;
      push("fine_gather_coarse", [=](cudaStream_t st) {
        return fine_gather_coarse(tok_, 512, B_, L_, cmb.b_ids, cmb.i_ids, cmb.j_ids, cmb.m_total, Mc, cin_, st);
      });
      conv("fine.down_proj", cin, 2, 1, Mcap, 256, 256, 128, 1, 1, true, nullptr, ACT_NONE, cproj, 128, 0,
           cm.m_total);
    }
    const size_t windows_step = steps.size();
    fine_windows(featf, img_f, featf + B * img_f, img_f);
    {
      conv("fine.merge_feat", win, 2, 1, Mcap * 25, 256, 256, 128, 1, 1, true, nullptr, ACT_NONE, ftok, 256, 0,
           cm.m_total + 2);
    }
    {
      const int rows = Mcap * 25;
      if (precision == 1) {   // bf16 shadow of the fine tokens (the encoder layers keep it current from here on)
        for (int side = 0; side < 2; ++side) {
          const float* src = ftok + static_cast<size_t>(side) * rows * 256;
          float* dst = ftokb + static_cast<size_t>(side) * rows * 256 / 2;
          const int* dr = cm.m_total + 2;
          push("to_bf16", [=](cudaStream_t st) { return rows_to_bf16(src, 256, dst, 256, rows, 128, dr, st); });
        }
      }
      const size_t s_tok = static_cast<size_t>(rows) * 256, s_qkv = static_cast<size_t>(rows) * 384,
                   s_c = static_cast<size_t>(rows) * 128, s_2c = static_cast<size_t>(rows) * 256;
      encoder_layer("fine.0", 128, ftok, ftok, fqkv, fqkv, fmsg, fmrg, fh1, fh2, 2, rows, cm.m_total + 2,
                    cm.m_total, true);
      encoder_layer("fine.1", 128, ftok, ftok + s_tok, fqkv, fqkv + s_qkv / tb, fmsg, fmrg, fh1, fh2, 1, rows,
                    cm.m_total + 2, cm.m_total, true);
      encoder_layer("fine.1", 128, ftok + s_tok, ftok, fqkv + s_qkv / tb, fqkv, fmsg + s_c / tb, at(fmrg, s_c),
                    at(fh1, s_2c), at(fh2, s_c), 1, rows, cm.m_total + 2, cm.m_total, true);
      CoarseMatchBuffers cmb = cm; float *f0 = ftok, *f1 = ftok + s_tok, *mk = mk1f, *ex = expec;
      const int Mc = Mcap; const float scale_f = static_cast<float>(H) / static_cast<float>(H2);
      push("fine_match", [=](cudaStream_t st) {
        return fine_match(f0, f1, 256, cmb.mkpts1_c, cmb.m_total, Mc, scale_f, mk, ex, st);
      });
    }
    if (rc != MFR_OK) return rc;

    // ---------------------------------------------------------------- shared map frame
    LaunchList paired = std::move(steps);
    steps = LaunchList();
    conv_count = kReservedLayers;   // the map encode runs once per scene, on its own: no SMs to leave free
    backbone(map_img, 1, fc, map_featf);
    coarse_tokens(fc, 1, map_tok);
    coarse_layer0(map_tok, 1);
    map_steps = std::move(steps);
    steps = LaunchList();
    conv_count = 0;
    const size_t half_img = static_cast<size_t>(B) * H * W;
    backbone(img + half_img, B, fc + half_c, featf + B * img_f);
    coarse_tokens(fc + half_c, B, tok + half_tok);
    {
      float *mt = map_tok, *mtb = map_tokb, *t0 = tok, *tb0 = tokb; const long long bytes = static_cast<long long>(L) * 512 * 4;
      const int nb = B;
      push("map_broadcast", [=](cudaStream_t st) {
        int rc = broadcast_copies(mt, bytes, t0, nb, st);
        if (rc == MFR_OK && mtb) rc = broadcast_copies(mtb, bytes / 2, tb0, nb, st);
        return rc;
      }, bf ? 2 : 1);
    }
    coarse_layer0(tok + half_tok, B);
    steps.append(paired, layer1_begin, windows_step);
    fine_windows(map_featf, 0, featf + B * img_f, img_f);
    steps.append(paired, windows_step + 1, paired.steps.size());
    shared_steps = std::move(steps);
    steps = std::move(paired);
    return rc;
  }

  // Copies `n` source images [n][src_h][src_w] into the engine frames dst [n][H][W]; the right/bottom remainder of a
  // frame stays zero: the reference's ConstantPad2d (matchers.py:41-46).
  int copy_frames(float* dst, const float* src, int n, int src_h, int src_w, cudaStream_t st) {
    if (src_h == H && src_w == W) {
      MFR_CUDA_CHECK(cudaMemcpyAsync(dst, src, static_cast<size_t>(n) * H * W * 4, cudaMemcpyDeviceToDevice, st));
      return MFR_OK;
    }
    for (int b = 0; b < n; ++b)
      MFR_CUDA_CHECK(cudaMemcpy2DAsync(dst + static_cast<size_t>(b) * H * W, static_cast<size_t>(W) * 4,
                                       src + static_cast<size_t>(b) * src_h * src_w, static_cast<size_t>(src_w) * 4,
                                       static_cast<size_t>(src_w) * 4, src_h, cudaMemcpyDeviceToDevice, st));
    return MFR_OK;
  }

  // Stages the batch into `img` (img0 == nullptr: the query half only). The pad of every frame in `img` is zero as
  // long as each call writes frames of the size of the previous call; a change of size clears the whole buffer.
  int stage(const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st) {
    if (src_h > H || src_w > W || src_h < 1 || src_w < 1) return MFR_ERR_ARG;
    const size_t half = static_cast<size_t>(B) * H * W;
    if ((src_h != H || src_w != W) && (src_h != last_src_h || src_w != last_src_w) && last_src_h > 0)
      MFR_CUDA_CHECK(cudaMemsetAsync(img, 0, 2 * half * 4, st));   // a smaller source than last time: clear the old pixels of the pad
    last_src_h = src_h; last_src_w = src_w;
    int rc = MFR_OK;
    if (img0) rc = copy_frames(img, img0, B, src_h, src_w, st);
    if (rc == MFR_OK) rc = copy_frames(img + half, img1, B, src_h, src_w, st);
    return rc;
  }

  // src images are [B][src_h][src_w] (src_h <= H, src_w <= W), zero-padded to the engine's [H][W] frame
  int forward(const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st) {
    if (!weights.complete()) {
      fprintf(stderr, "[mfr_b200] loftr forward before weights were loaded\n");
      return MFR_ERR_ARG;
    }
    int r = stage(img0, img1, src_h, src_w, st);
    if (r == MFR_OK) r = derived.rebuild(weights, st);
    if (r != MFR_OK) return r;
    return graph.launch(steps, st, use_graph, "loftr");
  }

  // Encodes one map image [src_h][src_w] (eagerly) into the map buffers, which forward_shared reads until the next
  // set_map or weight upload. The pixels of the frame outside the source stay zero, as in forward.
  int set_map(const float* img0, int src_h, int src_w, cudaStream_t st) {
    if (!weights.complete()) return MFR_ERR_ARG;
    if (src_h > H || src_w > W || src_h < 1 || src_w < 1) return MFR_ERR_ARG;
    map_gen = -1;
    int r = derived.rebuild(weights, st);
    if (r != MFR_OK) return r;
    if (src_h != H || src_w != W) MFR_CUDA_CHECK(cudaMemsetAsync(map_img, 0, static_cast<size_t>(H) * W * 4, st));
    r = copy_frames(map_img, img0, 1, src_h, src_w, st);
    if (r == MFR_OK) r = map_steps.run(st);
    if (r != MFR_OK) return r;
    map_src_h = src_h; map_src_w = src_w;
    map_gen = weights.generation;
    return MFR_OK;
  }

  // forward(map repeated B times, img1) without encoding the map again: the same bits in every output
  int forward_shared(const float* img1, int src_h, int src_w, cudaStream_t st) {
    if (!weights.complete() || map_gen != weights.generation || src_h != map_src_h || src_w != map_src_w) return MFR_ERR_ARG;
    const int r = stage(nullptr, img1, src_h, src_w, st);
    if (r != MFR_OK) return r;
    return shared_graph.launch(shared_steps, st, use_graph, "loftr");
  }

  // Steps [begin, end) of the paired forward list, eagerly, on the buffers as earlier calls left them
  int run_steps(int begin, int end, cudaStream_t st) {
    if (begin < 0 || end < begin || end > steps.size() || !weights.complete()) return MFR_ERR_ARG;
    const int r = derived.rebuild(weights, st);
    if (r != MFR_OK) return r;
    return steps.run(st, begin, end);
  }

  // eager run with a CUDA event pair around every step; ms[i] = device time of step i
  int profile(const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st, int max_steps,
              float* ms, double* flops, int* kinds, char* names) {
    const bool g = use_graph;
    use_graph = false;
    int r = forward(img0, img1, src_h, src_w, st);  // warm
    std::vector<float> t;
    if (r == MFR_OK) r = timed_run(steps, st, t);
    use_graph = g;
    if (r != MFR_OK) return -r;
    int m_total_h[4] = {0, 0, 0, 0};
    cudaMemcpy(m_total_h, cm.m_total, sizeof(m_total_h), cudaMemcpyDeviceToHost);
    for (int i = 0; i < steps.size() && i < max_steps; ++i) {
      const Step& s = steps.steps[i];
      ms[i] = t[i];
      flops[i] = s.dyn_rows ? s.flops * (static_cast<double>(m_total_h[s.dyn_rows - cm.m_total]) * s.dyn_images) : s.flops;
      kinds[i] = s.kind;
      strncpy(names + 32 * i, s.name.c_str(), 31);
      names[32 * i + 31] = 0;
    }
    return steps.size();
  }
};

// ---------------------------------------------------------------------------------------------
int loftr_create(int B, int H, int W, float thr, int border, float temperature, int precision, int reserved_sms,
                 LoftrEngine** out) {
  if (B < 1 || H % 8 || W % 8 || H < 32 || W < 32 || precision < 0 || precision > 2) return MFR_ERR_ARG;
  if (reserved_sms < 0 || reserved_sms >= conv_gemm_num_sms()) return MFR_ERR_ARG;
  auto* e = new LoftrEngine();
  e->B = B; e->H = H; e->W = W; e->thr = thr; e->border = border; e->temperature = temperature;
  e->precision = precision; e->reserved_sms = reserved_sms;
  const int rc = e->build();
  if (rc != MFR_OK) { delete e; return rc; }
  *out = e;
  return MFR_OK;
}
void loftr_destroy(LoftrEngine* e) { delete e; }
EngineCore& engine_core(LoftrEngine* e) { return *e; }
int loftr_forward(LoftrEngine* e, const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st) {
  return e->forward(img0, img1, src_h, src_w, st);
}
int loftr_set_map(LoftrEngine* e, const float* img0, int src_h, int src_w, cudaStream_t st) {
  return e->set_map(img0, src_h, src_w, st);
}
int loftr_forward_shared(LoftrEngine* e, const float* img1, int src_h, int src_w, cudaStream_t st) {
  return e->forward_shared(img1, src_h, src_w, st);
}
void loftr_outputs(LoftrEngine* e, mfr_loftr_outputs* o) {
  o->m_total = e->cm.m_total; o->m_offsets = e->cm.m_offsets; o->b_ids = e->cm.b_ids;
  o->i_ids = e->cm.i_ids; o->j_ids = e->cm.j_ids; o->mconf = e->cm.mconf;
  o->mkpts0_f = e->cm.mkpts0_c; o->mkpts1_f = e->mk1f; o->mkpts1_c = e->cm.mkpts1_c; o->expec_f = e->expec;
  o->capacity = e->Mcap;
}
int loftr_profile(LoftrEngine* e, const float* img0, const float* img1, int src_h, int src_w, cudaStream_t st,
                  int max_steps, float* ms, double* flops, int* kinds, char* names) {
  return e->profile(img0, img1, src_h, src_w, st, max_steps, ms, flops, kinds, names);
}
int loftr_run_steps(LoftrEngine* e, int begin, int end, cudaStream_t st) { return e->run_steps(begin, end, st); }

}  // namespace mfr
