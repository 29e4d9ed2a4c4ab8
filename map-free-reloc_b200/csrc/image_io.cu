// Input path of the matchers on the GPU (SURVEY §8(f) rank 1): JPEG decode (the arithmetic of cv2.imread, jpeg.cuh) +
// the resize / normalise step of the reference's loaders
//   read_image      etc/feature_matching_baselines/SuperGlue/models/utils.py:263-285   gray, cv2.resize, / 255
//   read_color_image lib/datasets/utils.py:58-75                                        RGB uint8 cv2.resize, / 255, CHW
// cv2.resize(INTER_LINEAR) is restated for both of its code paths: float32 images (bilinear weights in fp32, horizontal
// pass first) and uint8 images (11-bit fixed-point weights, OpenCV's two-stage rounding), so that the resized pixels are
// the ones the reference feeds its networks. 16-bit depth PNGs (read_depth_image, lib/datasets/utils.py:77-81) are
// decoded here too (png.cuh). Inflate runs one warp per file; on an H100 a batch of 64 depth maps decodes faster than
// OpenCV on 8 host threads, a single file slower than one (DESIGN §3.8, §6).
//
// JPEG: a host marker parser validates each file and builds its descriptor (jpeg::Desc); one pinned staging buffer
// carries descriptors, restart-interval offsets and entropy-coded bytes to the device in one copy; three kernels follow:
// entropy decode (one thread per decode unit: the image, or one restart interval), dequantise + ISLOW IDCT (one thread
// per block), upsample + colour + Exif orientation (one thread per output pixel).
#include <algorithm>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "jpeg.cuh"
#include "png.cuh"

namespace mfr {

namespace {

// source coordinate of destination pixel d (cv2: fx = (dx + 0.5) * scale - 0.5, clamped like resizeGeneric's tables)
__device__ __forceinline__ void src_coord(int d, double scale, int ssize, int& s0, float& f) {
  float fx = static_cast<float>((d + 0.5) * scale - 0.5);
  int sx = static_cast<int>(floorf(fx));
  fx -= sx;
  if (sx < 0) { fx = 0.f; sx = 0; }
  if (sx >= ssize - 1) { fx = 0.f; sx = ssize - 1; }
  s0 = sx; f = fx;
}

// float path: dst = ((1-fy) * ((1-fx) S00 + fx S01) + fy * ((1-fx) S10 + fx S11)) * out_scale, SRC = float or uint8 (converted first)
template <typename SRC>
__global__ void resize_linear_f32_kernel(const SRC* __restrict__ src, int sw, int sh, long long src_stride, int channels,
                                         float* __restrict__ dst, int dw, int dh, double sx, double sy, float out_scale, int chw) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  int x0, y0; float fx, fy;
  src_coord(x, sx, sw, x0, fx);
  src_coord(y, sy, sh, y0, fy);
  const int x1 = min(x0 + 1, sw - 1), y1 = min(y0 + 1, sh - 1);
  for (int c = 0; c < channels; ++c) {
    const float s00 = static_cast<float>(src[y0 * src_stride + x0 * channels + c]), s01 = static_cast<float>(src[y0 * src_stride + x1 * channels + c]);
    const float s10 = static_cast<float>(src[y1 * src_stride + x0 * channels + c]), s11 = static_cast<float>(src[y1 * src_stride + x1 * channels + c]);
    const float r0 = __fadd_rn(__fmul_rn(s00, 1.f - fx), __fmul_rn(s01, fx));      // HResizeLinear: S[x] * a0 + S[x+1] * a1
    const float r1 = __fadd_rn(__fmul_rn(s10, 1.f - fx), __fmul_rn(s11, fx));
    const float v = __fadd_rn(__fmul_rn(r0, 1.f - fy), __fmul_rn(r1, fy));        // VResizeLinear: S0 * b0 + S1 * b1
    const size_t o = chw ? (static_cast<size_t>(c) * dh + y) * dw + x : (static_cast<size_t>(y) * dw + x) * channels + c;
    dst[o] = v * out_scale;
  }
}

// uint8 path (cv2.resize on uint8): INTER_RESIZE_COEF_BITS = 11 fixed-point weights, rows kept as int (x 2048), vertical
// pass ((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2, saturated to uint8; then float * out_scale
__global__ void resize_linear_u8_kernel(const unsigned char* __restrict__ src, int sw, int sh, long long src_stride, int channels,
                                        float* __restrict__ dst, int dw, int dh, double sx, double sy, float out_scale, int chw) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= dw) return;
  int x0, y0; float fx, fy;
  src_coord(x, sx, sw, x0, fx);
  src_coord(y, sy, sh, y0, fy);
  const int x1 = min(x0 + 1, sw - 1), y1 = min(y0 + 1, sh - 1);
  auto coef = [](float v) { return static_cast<int>(max(-32768, min(32767, __float2int_rn(v * 2048.f)))); };   // saturate_cast<short>(cvRound)
  const int a0 = coef(1.f - fx), a1 = coef(fx), b0 = coef(1.f - fy), b1 = coef(fy);
  for (int c = 0; c < channels; ++c) {
    const int r0 = src[y0 * src_stride + x0 * channels + c] * a0 + src[y0 * src_stride + x1 * channels + c] * a1;
    const int r1 = src[y1 * src_stride + x0 * channels + c] * a0 + src[y1 * src_stride + x1 * channels + c] * a1;
    int v = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
    v = max(0, min(255, v));
    const size_t o = chw ? (static_cast<size_t>(c) * dh + y) * dw + x : (static_cast<size_t>(y) * dw + x) * channels + c;
    dst[o] = static_cast<float>(v) * out_scale;
  }
}

}  // namespace

// mode 0: float path on a float32 source; 1: float path on a uint8 source (image.astype('float32') then resize: read_image with
// resize_float=True); 2: uint8 fixed-point path (cv2.resize on uint8, then float). dst = resized * out_scale.
int resize_linear(const void* src, int src_is_u8, int sw, int sh, long long src_stride, int channels, float* dst, int dw, int dh,
                  int mode, float out_scale, int chw, cudaStream_t st) {
  if (!src || !dst || sw < 1 || sh < 1 || dw < 1 || dh < 1 || channels < 1 || channels > 4) return MFR_ERR_ARG;
  const double sx = static_cast<double>(sw) / dw, sy = static_cast<double>(sh) / dh;
  const dim3 grid((dw + 127) / 128, dh), block(128);
  if (mode == 2) {
    if (!src_is_u8) return MFR_ERR_ARG;
    resize_linear_u8_kernel<<<grid, block, 0, st>>>(static_cast<const unsigned char*>(src), sw, sh, src_stride, channels, dst, dw, dh, sx, sy, out_scale, chw);
  } else if (src_is_u8) {
    resize_linear_f32_kernel<unsigned char><<<grid, block, 0, st>>>(static_cast<const unsigned char*>(src), sw, sh, src_stride, channels, dst, dw, dh, sx, sy, out_scale, chw);
  } else {
    resize_linear_f32_kernel<float><<<grid, block, 0, st>>>(static_cast<const float*>(src), sw, sh, src_stride, channels, dst, dw, dh, sx, sy, out_scale, chw);
  }
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

// ============================================================================================ JPEG
namespace {

using jpeg::Desc;
using jpeg::Huff;

const uint8_t kNaturalHost[jpeg::kNaturalLen] = MFR_JPEG_NATURAL_ORDER;
__constant__ uint8_t c_natural[jpeg::kNaturalLen] = MFR_JPEG_NATURAL_ORDER;

// One parsed file: its descriptor (offsets relative to the file), the entropy-coded byte range and the unit offsets.
struct Parsed {
  Desc d;
  size_t ent_begin = 0, ent_len = 0;
  std::vector<uint32_t> units;     // per decode unit its byte range (start, end) in the entropy-coded bytes
  long long samples = 0;           // coefficient / sample count of all planes
};

struct RawHuff {
  bool defined = false;
  uint8_t counts[17] = {};
  uint8_t vals[256] = {};
  int n = 0;
};

unsigned be16(const uint8_t* p) { return (static_cast<unsigned>(p[0]) << 8) | p[1]; }

// canonical codes (T.81 C.2) -> lookahead LUT + maxcode / valoff; false if the counts over-subscribe the code space
bool build_huff(const RawHuff& r, Huff& t) {
  memset(&t, 0, sizeof(t));
  int code = 0, k = 0;
  for (int l = 1; l <= 16; ++l) {
    const int n = r.counts[l];
    t.valoff[l] = k - code;
    t.maxcode[l] = n ? code + n - 1 : -1;
    if (code + n > (1 << l)) return false;
    for (int i = 0; i < n; ++i, ++k, ++code) {
      t.vals[k] = r.vals[k];
      if (l <= jpeg::kLutBits) {
        const int shift = jpeg::kLutBits - l;
        for (int f = 0; f < (1 << shift); ++f) t.lut[(code << shift) | f] = static_cast<uint16_t>((l << 8) | r.vals[k]);
      }
    }
    code <<= 1;
  }
  t.maxcode[17] = 0x7FFFFFFF;
  return true;
}

// Exif Orientation (tag 0x0112 of IFD0) of an APP1 payload that starts with "Exif\0\0"; 1 when absent or malformed
int exif_orientation(const uint8_t* p, size_t n) {
  if (n < 14 || memcmp(p, "Exif\0\0", 6) != 0) return 1;
  const uint8_t* t = p + 6;
  const size_t tn = n - 6;
  bool le;
  if (t[0] == 'I' && t[1] == 'I') le = true;
  else if (t[0] == 'M' && t[1] == 'M') le = false;
  else return 1;
  auto u16 = [&](size_t o) -> unsigned { return le ? t[o] | (t[o + 1] << 8) : (t[o] << 8) | t[o + 1]; };
  auto u32 = [&](size_t o) -> size_t { return le ? (size_t)u16(o) | ((size_t)u16(o + 2) << 16) : ((size_t)u16(o) << 16) | u16(o + 2); };
  if (u16(2) != 42) return 1;
  const size_t ifd = u32(4);
  if (ifd + 2 > tn) return 1;
  const unsigned cnt = u16(ifd);
  for (unsigned i = 0; i < cnt; ++i) {
    const size_t e = ifd + 2 + 12 * static_cast<size_t>(i);
    if (e + 12 > tn) return 1;
    if (u16(e) == 0x0112) {
      const unsigned v = u16(e + 8);
      return v >= 1 && v <= 8 ? static_cast<int>(v) : 1;
    }
  }
  return 1;
}

// Parses and validates one file. MFR_OK: `out` describes a file the kernels decode; MFR_ERR_UNSUPPORTED: a valid file
// outside the supported set (progressive, arithmetic, lossless, 12-bit, 4:4:0 / 4:1:1, CMYK, RGB-coded, multi-scan);
// MFR_ERR_ARG: malformed headers (lengths, tables, geometry) or entropy data whose restart markers disagree with them.
int parse_jpeg(const uint8_t* data, size_t len, int rgb, Parsed& out) {
  if (!data || len < 4 || len > 0xFFFFFFFFull || data[0] != 0xFF || data[1] != 0xD8) return MFR_ERR_ARG;
  Desc& d = out.d;
  memset(&d, 0, sizeof(d));
  d.orient = 1;
  d.rgb = rgb;
  RawHuff dht[2][4];
  int qt[4][64];
  bool qdef[4] = {false, false, false, false};
  int comp_id[3] = {0, 0, 0}, comp_tq[3] = {0, 0, 0}, comp_hs[3] = {0, 0, 0}, comp_vs[3] = {0, 0, 0};
  bool sof = false, jfif = false, adobe = false, exif_seen = false;
  int adobe_transform = -1;
  size_t pos = 2;
  for (;;) {
    if (pos + 2 > len || data[pos] != 0xFF) return MFR_ERR_ARG;
    while (pos < len && data[pos] == 0xFF) ++pos;          // fill bytes
    if (pos >= len) return MFR_ERR_ARG;
    const int m = data[pos++];
    if (m == 0xD8 || m == 0xD9 || m == 0x01 || (m >= 0xD0 && m <= 0xD7) || m == 0x00) return MFR_ERR_ARG;
    if (pos + 2 > len) return MFR_ERR_ARG;
    const size_t L = be16(data + pos);
    if (L < 2 || pos + L > len) return MFR_ERR_ARG;
    const uint8_t* seg = data + pos + 2;
    const size_t n = L - 2;
    if (m == 0xC0 || m == 0xC1) {                          // SOF0 / SOF1: Huffman, sequential
      if (sof || n < 6) return MFR_ERR_ARG;
      sof = true;
      if (seg[0] != 8) return MFR_ERR_UNSUPPORTED;          // 12-bit
      d.height = static_cast<int>(be16(seg + 1));
      d.width = static_cast<int>(be16(seg + 3));
      d.ncomp = seg[5];
      if (d.height == 0) return MFR_ERR_UNSUPPORTED;        // height from a DNL marker
      if (d.width == 0 || d.ncomp == 0) return MFR_ERR_ARG;
      if (d.ncomp != 1 && d.ncomp != 3) return MFR_ERR_UNSUPPORTED;
      if (n != 6 + 3 * static_cast<size_t>(d.ncomp)) return MFR_ERR_ARG;
      for (int c = 0; c < d.ncomp; ++c) {
        comp_id[c] = seg[6 + 3 * c];
        comp_hs[c] = seg[7 + 3 * c] >> 4;
        comp_vs[c] = seg[7 + 3 * c] & 15;
        comp_tq[c] = seg[8 + 3 * c];
        if (comp_hs[c] < 1 || comp_hs[c] > 4 || comp_vs[c] < 1 || comp_vs[c] > 4 || comp_tq[c] > 3) return MFR_ERR_ARG;
        for (int e = 0; e < c; ++e)
          if (comp_id[e] == comp_id[c]) return MFR_ERR_ARG;
      }
    } else if (m >= 0xC2 && m <= 0xCF && m != 0xC4) {   // progressive, lossless, hierarchical, arithmetic (DAC too)
      return MFR_ERR_UNSUPPORTED;
    } else if (m == 0xC4) {                                 // DHT: one or more tables
      size_t o = 0;
      while (o < n) {
        if (o + 17 > n) return MFR_ERR_ARG;
        const int tc = seg[o] >> 4, th = seg[o] & 15;
        if (tc > 1 || th > 3) return MFR_ERR_ARG;
        RawHuff& r = dht[tc][th];
        r.n = 0;
        for (int l = 1; l <= 16; ++l) { r.counts[l] = seg[o + l]; r.n += r.counts[l]; }
        if (r.n > 256 || o + 17 + r.n > n) return MFR_ERR_ARG;   // incomplete table
        memcpy(r.vals, seg + o + 17, r.n);
        if (tc == 0)
          for (int i = 0; i < r.n; ++i)
            if (r.vals[i] > 15) return MFR_ERR_ARG;         // DC categories of at most 15 bits (libjpeg's limit)
        Huff probe;
        if (!build_huff(r, probe)) return MFR_ERR_ARG;
        r.defined = true;
        o += 17 + r.n;
      }
    } else if (m == 0xDB) {                                 // DQT: 8- or 16-bit tables, zig-zag order
      size_t o = 0;
      while (o < n) {
        const int pq = seg[o] >> 4, tq = seg[o] & 15;
        if (pq > 1 || tq > 3 || o + 1 + 64 * (pq + 1) > n) return MFR_ERR_ARG;
        for (int k = 0; k < 64; ++k) {
          const unsigned v = pq ? be16(seg + o + 1 + 2 * k) : seg[o + 1 + k];
          qt[tq][kNaturalHost[k]] = static_cast<int16_t>(v);   // libjpeg's ISLOW_MULT_TYPE is 16-bit
        }
        qdef[tq] = true;
        o += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xDD) {                                 // DRI
      if (n != 2) return MFR_ERR_ARG;
      d.restart = static_cast<int>(be16(seg));
    } else if (m == 0xE0) {
      if (n >= 5 && memcmp(seg, "JFIF\0", 5) == 0) jfif = true;
    } else if (m == 0xE1) {
      if (!exif_seen && n >= 6 && memcmp(seg, "Exif\0\0", 6) == 0) { exif_seen = true; d.orient = exif_orientation(seg, n); }
    } else if (m == 0xEE) {
      if (n >= 12 && memcmp(seg, "Adobe", 5) == 0) { adobe = true; adobe_transform = seg[11]; }
    } else if (m == 0xDA) {                                 // SOS: the one scan
      if (!sof || n < 1) return MFR_ERR_ARG;
      const int ns = seg[0];
      if (n != 4 + 2 * static_cast<size_t>(ns) || ns < 1 || ns > 4) return MFR_ERR_ARG;
      if (ns != d.ncomp) return MFR_ERR_UNSUPPORTED;        // one component per scan: a multi-scan file
      for (int c = 0; c < ns; ++c)
        if (seg[1 + 2 * c] != comp_id[c]) return MFR_ERR_UNSUPPORTED;   // scan order other than frame order
      const uint8_t* tail = seg + 1 + 2 * ns;
      if (tail[0] != 0 || tail[1] != 63 || tail[2] != 0) return MFR_ERR_UNSUPPORTED;   // not a full sequential scan
      // colour space as libjpeg infers it: RGB-coded three-component files are not converted from YCbCr
      if (d.ncomp == 3 && !jfif &&
          ((adobe && adobe_transform == 0) || (!adobe && comp_id[0] == 'R' && comp_id[1] == 'G' && comp_id[2] == 'B')))
        return MFR_ERR_UNSUPPORTED;
      // geometry
      if (d.ncomp == 1) {
        comp_hs[0] = comp_vs[0] = 1;                        // a one-component scan is not interleaved
      } else {
        const bool y_ok = (comp_hs[0] == 1 && comp_vs[0] == 1) || (comp_hs[0] == 2 && comp_vs[0] == 1) ||
                          (comp_hs[0] == 2 && comp_vs[0] == 2);
        if (!y_ok || comp_hs[1] != 1 || comp_vs[1] != 1 || comp_hs[2] != 1 || comp_vs[2] != 1) return MFR_ERR_UNSUPPORTED;
      }
      d.hmax = comp_hs[0];
      d.vmax = comp_vs[0];
      d.mcus_x = (d.width + 8 * d.hmax - 1) / (8 * d.hmax);
      d.mcus_y = (d.height + 8 * d.vmax - 1) / (8 * d.vmax);
      int tmap[2][4];
      for (auto& r : tmap) for (int& v : r) v = -1;
      long long coef = 0;
      d.n_blocks = 0;
      for (int c = 0; c < d.ncomp; ++c) {
        jpeg::Comp& cp = d.comp[c];
        cp.h = comp_hs[c]; cp.v = comp_vs[c];
        cp.bw = d.mcus_x * cp.h; cp.bh = d.mcus_y * cp.v;
        cp.dw = (d.width * cp.h + d.hmax - 1) / d.hmax;
        cp.dh = (d.height * cp.v + d.vmax - 1) / d.vmax;
        cp.coef = coef;
        cp.plane = coef;
        coef += static_cast<long long>(cp.bw) * cp.bh * 64;
        d.n_blocks += cp.bw * cp.bh;
        if (!qdef[comp_tq[c]]) return MFR_ERR_ARG;
        memcpy(d.qt[c], qt[comp_tq[c]], sizeof(d.qt[c]));
        const int td = seg[2 + 2 * c] >> 4, ta = seg[2 + 2 * c] & 15;
        if (td > 3 || ta > 3 || !dht[0][td].defined || !dht[1][ta].defined) return MFR_ERR_ARG;   // table missing
        for (int k = 0; k < 2; ++k) {
          const int id = k ? ta : td;
          if (tmap[k][id] < 0) {
            tmap[k][id] = d.n_tbl;
            build_huff(dht[k][id], d.tbl[d.n_tbl++]);
          }
        }
        cp.dc = tmap[0][td];
        cp.ac = tmap[1][ta];
      }
      out.samples = coef;
      // entropy-coded data: up to the first marker other than RSTn; restart intervals split at RSTn, each unit a byte
      // range (start, end) relative to `begin`
      const size_t begin = pos + L;
      out.units.clear();
      out.units.push_back(0);
      size_t q = begin;
      for (;;) {
        if (q + 1 >= len) { q = len; break; }                // no terminating marker: the data runs to the end
        if (data[q] != 0xFF) { ++q; continue; }
        const uint8_t nx = data[q + 1];
        if (nx == 0x00) { q += 2; continue; }
        if (nx == 0xFF) { ++q; continue; }
        if (nx >= 0xD0 && nx <= 0xD7) {
          if (!d.restart) return MFR_ERR_ARG;
          out.units.push_back(static_cast<uint32_t>(q - begin));
          out.units.push_back(static_cast<uint32_t>(q + 2 - begin));
          q += 2;
          continue;
        }
        break;
      }
      out.ent_begin = begin;
      out.ent_len = q - begin;
      out.units.push_back(static_cast<uint32_t>(q - begin));
      const long long total = static_cast<long long>(d.mcus_x) * d.mcus_y;
      const long long expect = d.restart ? (total + d.restart - 1) / d.restart : 1;
      if (static_cast<long long>(out.units.size()) != 2 * expect) return MFR_ERR_ARG;   // restart markers vs geometry
      d.n_units = static_cast<int>(expect);
      const bool swap = d.orient >= 5;
      d.out_w = swap ? d.height : d.width;
      d.out_h = swap ? d.width : d.height;
      d.status = MFR_OK;
      return MFR_OK;
    }
    // APPn other than the above, COM, and anything else with a length: skipped
    pos += L;
  }
}

// ------------------------------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(64) jpeg_entropy_kernel(const Desc* __restrict__ descs, const uint32_t* __restrict__ units,
                                                          const uint8_t* __restrict__ data, int16_t* __restrict__ coef,
                                                          int* __restrict__ status) {
  __shared__ Huff tbl[jpeg::kMaxTables];
  __shared__ uint8_t nat[jpeg::kNaturalLen];
  const Desc& d = descs[blockIdx.y];
  if (d.status != MFR_OK || blockIdx.x * blockDim.x >= static_cast<unsigned>(d.n_units)) return;
  const uint32_t* src = reinterpret_cast<const uint32_t*>(d.tbl);
  uint32_t* dst = reinterpret_cast<uint32_t*>(tbl);
  const int words = d.n_tbl * static_cast<int>(sizeof(Huff) / 4);
  for (int i = threadIdx.x; i < words; i += blockDim.x) dst[i] = src[i];
  for (int i = threadIdx.x; i < jpeg::kNaturalLen; i += blockDim.x) nat[i] = c_natural[i];
  __syncthreads();
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= d.n_units) return;
  if (jpeg::decode_unit(d, tbl, nat, data + d.data, units + d.units, u, coef)) status[blockIdx.y] = MFR_ERR_ARG;
}

__global__ void __launch_bounds__(128) jpeg_idct_kernel(const Desc* __restrict__ descs, const int16_t* __restrict__ coef,
                                                        uint8_t* __restrict__ planes) {
  const Desc& d = descs[blockIdx.y];
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (d.status != MFR_OK || b >= d.n_blocks) return;
  int c = 0, bb = b;
  while (bb >= d.comp[c].bw * d.comp[c].bh) { bb -= d.comp[c].bw * d.comp[c].bh; ++c; }
  const jpeg::Comp& cp = d.comp[c];
  const int bx = bb % cp.bw, by = bb / cp.bw, stride = cp.bw * 8;
  jpeg::idct_block(coef + cp.coef + 64LL * bb, d.qt[c], planes + cp.plane + static_cast<long long>(by) * 8 * stride + bx * 8, stride);
}

__global__ void __launch_bounds__(256) jpeg_pixel_kernel(const Desc* __restrict__ descs, const uint8_t* __restrict__ planes) {
  const Desc& d = descs[blockIdx.y];
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (d.status != MFR_OK || p >= static_cast<long long>(d.out_w) * d.out_h) return;
  const int ox = static_cast<int>(p % d.out_w), oy = static_cast<int>(p / d.out_w);
  uint8_t px[3];
  jpeg::pixel(d, planes, ox, oy, px);
  if (d.rgb) { d.dst[3 * p] = px[0]; d.dst[3 * p + 1] = px[1]; d.dst[3 * p + 2] = px[2]; }
  else d.dst[p] = px[0];
}

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

}  // namespace

// ------------------------------------------------------------------------------------------ staging (JPEG and PNG)
// One batch's inputs travel in one pinned buffer and one host-to-device copy. `copied` tells the host when it may
// refill the pinned buffer, `done` tells the next batch's stream when the device buffers are free again.
struct Staging {
  size_t bytes = 0;
  unsigned char* h = nullptr;   // pinned
  unsigned char* d = nullptr;
  cudaEvent_t copied = nullptr, done = nullptr;
};

bool staging_create(Staging& s, size_t bytes) {
  s.bytes = bytes;
  return cudaHostAlloc(&s.h, bytes, cudaHostAllocDefault) == cudaSuccess && cudaMalloc(&s.d, bytes) == cudaSuccess &&
         cudaEventCreateWithFlags(&s.copied, cudaEventDisableTiming) == cudaSuccess &&
         cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming) == cudaSuccess;
}

void staging_destroy(Staging& s) {
  if (s.done) cudaEventSynchronize(s.done);
  if (s.copied) cudaEventDestroy(s.copied);
  if (s.done) cudaEventDestroy(s.done);
  if (s.h) cudaFreeHost(s.h);
  cudaFree(s.d);
  s = Staging();
}

// before the host writes s.h: the previous call's staging has reached the device
int staging_acquire(Staging& s) {
  MFR_CUDA_CHECK(cudaEventSynchronize(s.copied));
  return MFR_OK;
}

// the first `total` bytes of s.h to s.d on `st`, once the previous call's kernels are done with the device buffers
int staging_upload(Staging& s, size_t total, cudaStream_t st) {
  MFR_CUDA_CHECK(cudaStreamWaitEvent(st, s.done, 0));
  MFR_CUDA_CHECK(cudaMemcpyAsync(s.d, s.h, total, cudaMemcpyHostToDevice, st));
  MFR_CUDA_CHECK(cudaEventRecord(s.copied, st));
  return MFR_OK;
}

// after the call's last kernel
int staging_release(Staging& s, cudaStream_t st) {
  MFR_CUDA_CHECK(cudaEventRecord(s.done, st));
  return MFR_OK;
}

// ------------------------------------------------------------------------------------------ JPEG decoder
struct JpegDecoder {
  int max_images = 0;
  long long max_bytes = 0, sample_cap = 0, unit_cap = 0;
  Staging stage;
  int16_t* coef = nullptr;
  uint8_t* planes = nullptr;
  std::vector<Parsed> parsed;
};

void jpeg_decoder_destroy(JpegDecoder* dec) {
  if (!dec) return;
  staging_destroy(dec->stage);
  cudaFree(dec->coef);
  cudaFree(dec->planes);
  delete dec;
}

int jpeg_decoder_create(int max_images, long long max_bytes, long long max_pixels, JpegDecoder** out) {
  if (!out || max_images < 1 || max_images > 65535 || max_bytes < 1 || max_pixels < 1) return MFR_ERR_ARG;
  *out = nullptr;
  JpegDecoder* dec = new JpegDecoder();
  dec->max_images = max_images;
  dec->max_bytes = max_bytes;
  dec->sample_cap = 3 * max_pixels;
  dec->unit_cap = 2 * (dec->sample_cap / 64 + max_images);
  const size_t stage_bytes = align_up(static_cast<size_t>(max_images) * sizeof(Desc), 256) + align_up(4ull * max_images, 256) +
                             align_up(4ull * dec->unit_cap, 256) + static_cast<size_t>(max_bytes);
  bool ok = staging_create(dec->stage, stage_bytes) &&
            cudaMalloc(&dec->coef, 2 * dec->sample_cap) == cudaSuccess &&
            cudaMalloc(&dec->planes, dec->sample_cap) == cudaSuccess;
  if (!ok) {
    jpeg_decoder_destroy(dec);
    return MFR_ERR_CUDA;
  }
  dec->parsed.resize(max_images);
  *out = dec;
  return MFR_OK;
}

int jpeg_info(const unsigned char* data, size_t length, int* width, int* height, int* components) {
  Parsed p;
  const int rc = parse_jpeg(data, length, 0, p);
  if (rc != MFR_OK) return rc;
  *width = p.d.out_w; *height = p.d.out_h; *components = p.d.ncomp;
  return MFR_OK;
}

int jpeg_decode_batch(JpegDecoder* dec, const unsigned char* const* data, const long long* lengths, int n, int rgb,
                      unsigned char* const* dst, int* status, cudaStream_t st) {
  if (!dec || n < 0 || n > dec->max_images || (n > 0 && (!data || !lengths || !dst || !status))) return MFR_ERR_ARG;
  if (n == 0) return MFR_OK;
  long long bytes = 0, samples = 0, units = 0;
  int max_units = 0, max_blocks = 0;
  long long max_px = 0;
  for (int i = 0; i < n; ++i) {
    Parsed& p = dec->parsed[i];
    int rc = (data[i] && lengths[i] > 0) ? parse_jpeg(data[i], static_cast<size_t>(lengths[i]), rgb ? 1 : 0, p) : MFR_ERR_ARG;
    if (rc == MFR_OK && !dst[i]) rc = MFR_ERR_ARG;
    if (rc != MFR_OK) { memset(&p.d, 0, sizeof(Desc)); p.d.status = rc; p.ent_len = 0; p.units.clear(); p.samples = 0; continue; }
    p.d.dst = dst[i];
    p.d.data = bytes;
    p.d.units = units;
    for (int c = 0; c < p.d.ncomp; ++c) { p.d.comp[c].coef += samples; p.d.comp[c].plane += samples; }
    bytes += static_cast<long long>(p.ent_len);
    samples += p.samples;
    units += static_cast<long long>(p.units.size());
    max_units = std::max(max_units, p.d.n_units);
    max_blocks = std::max(max_blocks, p.d.n_blocks);
    max_px = std::max(max_px, static_cast<long long>(p.d.out_w) * p.d.out_h);
  }
  if (bytes > dec->max_bytes || samples > dec->sample_cap || units > dec->unit_cap) return MFR_ERR_ARG;   // over capacity
  // staging layout: descriptors | initial statuses | unit offsets | entropy-coded bytes
  const size_t off_status = align_up(static_cast<size_t>(n) * sizeof(Desc), 256);
  const size_t off_units = off_status + align_up(4ull * n, 256);
  const size_t off_data = off_units + align_up(4ull * units, 256);
  const size_t total = off_data + static_cast<size_t>(bytes);
  int rc = staging_acquire(dec->stage);
  if (rc != MFR_OK) return rc;
  unsigned char* h = dec->stage.h;
  Desc* hd = reinterpret_cast<Desc*>(h);
  int* hs = reinterpret_cast<int*>(h + off_status);
  uint32_t* hu = reinterpret_cast<uint32_t*>(h + off_units);
  for (int i = 0; i < n; ++i) {
    const Parsed& p = dec->parsed[i];
    hd[i] = p.d;
    hs[i] = p.d.status;
    if (p.d.status != MFR_OK) continue;
    memcpy(hu + p.d.units, p.units.data(), 4 * p.units.size());
    memcpy(h + off_data + p.d.data, data[i] + p.ent_begin, p.ent_len);
  }
  rc = staging_upload(dec->stage, total, st);
  if (rc != MFR_OK) return rc;
  const unsigned char* ds = dec->stage.d;
  const Desc* dd = reinterpret_cast<const Desc*>(ds);
  MFR_CUDA_CHECK(cudaMemcpyAsync(status, ds + off_status, 4ull * n, cudaMemcpyDeviceToDevice, st));
  if (samples > 0) {
    MFR_CUDA_CHECK(cudaMemsetAsync(dec->coef, 0, 2ull * samples, st));
    jpeg_entropy_kernel<<<dim3((max_units + 63) / 64, n), 64, 0, st>>>(
        dd, reinterpret_cast<const uint32_t*>(ds + off_units), ds + off_data, dec->coef, status);
    jpeg_idct_kernel<<<dim3((max_blocks + 127) / 128, n), 128, 0, st>>>(dd, dec->coef, dec->planes);
    jpeg_pixel_kernel<<<dim3(static_cast<unsigned>((max_px + 255) / 256), n), 256, 0, st>>>(dd, dec->planes);
    MFR_CUDA_CHECK(cudaGetLastError());
  }
  return staging_release(dec->stage, st);
}

void jpeg_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* status) {
  Parsed p;
  for (int i = 0; i < n; ++i) {
    status[i] = (data[i] && lengths[i] > 0) ? parse_jpeg(data[i], static_cast<size_t>(lengths[i]), 0, p) : MFR_ERR_ARG;
    width[i] = status[i] == MFR_OK ? p.d.out_w : 0;
    height[i] = status[i] == MFR_OK ? p.d.out_h : 0;
  }
}

// One file on the current device through a process-wide decoder per device, grown when a file does not fit; blocks
// until the decode is done so that the image's status can be returned.
int jpeg_decode(const unsigned char* data, size_t length, int rgb, unsigned char* dst, int width, int height, cudaStream_t st) {
  Parsed p;
  int rc = parse_jpeg(data, length, rgb ? 1 : 0, p);
  if (rc != MFR_OK) return rc;
  if (p.d.out_w != width || p.d.out_h != height) return MFR_ERR_ARG;
  struct Shared {
    JpegDecoder* dec = nullptr;
    int* status = nullptr;
    int* h_status = nullptr;
  };
  static std::mutex mu;
  static std::map<int, Shared> shared;
  int dev = 0;
  MFR_CUDA_CHECK(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  Shared& s = shared[dev];
  if (!s.status) {
    MFR_CUDA_CHECK(cudaMalloc(&s.status, sizeof(int)));
    MFR_CUDA_CHECK(cudaHostAlloc(&s.h_status, sizeof(int), cudaHostAllocDefault));
  }
  const long long px = (p.samples + 2) / 3 + 1;
  if (!s.dec || static_cast<long long>(length) > s.dec->max_bytes || p.samples > s.dec->sample_cap ||
      static_cast<long long>(p.units.size()) > s.dec->unit_cap) {
    jpeg_decoder_destroy(s.dec);
    s.dec = nullptr;
    rc = jpeg_decoder_create(1, std::max<long long>(static_cast<long long>(length), 1 << 20), std::max<long long>(px, 1 << 20), &s.dec);
    if (rc != MFR_OK) return rc;
  }
  const long long len = static_cast<long long>(length);
  rc = jpeg_decode_batch(s.dec, &data, &len, 1, rgb, &dst, s.status, st);
  if (rc != MFR_OK) return rc;
  MFR_CUDA_CHECK(cudaMemcpyAsync(s.h_status, s.status, sizeof(int), cudaMemcpyDeviceToHost, st));
  MFR_CUDA_CHECK(cudaStreamSynchronize(st));
  return *s.h_status;
}

// The same arithmetic serially on the CPU (test hook): dst [height][width] or [height][width][3], host memory.
int jpeg_host_decode(const unsigned char* data, size_t length, int rgb, unsigned char* dst, int width, int height) {
  Parsed p;
  const int rc = parse_jpeg(data, length, rgb ? 1 : 0, p);
  if (rc != MFR_OK) return rc;
  if (p.d.out_w != width || p.d.out_h != height) return MFR_ERR_ARG;
  const Desc& d = p.d;
  std::vector<int16_t> coef(p.samples, 0);
  std::vector<uint8_t> planes(p.samples, 0);
  const uint8_t* ent = data + p.ent_begin;
  for (int u = 0; u < d.n_units; ++u)
    if (jpeg::decode_unit(d, d.tbl, kNaturalHost, ent, p.units.data(), u, coef.data())) return MFR_ERR_ARG;
  for (int c = 0; c < d.ncomp; ++c) {
    const jpeg::Comp& cp = d.comp[c];
    for (int by = 0; by < cp.bh; ++by)
      for (int bx = 0; bx < cp.bw; ++bx)
        jpeg::idct_block(coef.data() + cp.coef + 64LL * (static_cast<long long>(by) * cp.bw + bx), d.qt[c],
                         planes.data() + cp.plane + static_cast<long long>(by) * 8 * cp.bw * 8 + bx * 8, cp.bw * 8);
  }
  const int ch = rgb ? 3 : 1;
  for (int oy = 0; oy < d.out_h; ++oy)
    for (int ox = 0; ox < d.out_w; ++ox) {
      uint8_t px[3];
      jpeg::pixel(d, planes.data(), ox, oy, px);
      memcpy(dst + (static_cast<size_t>(oy) * d.out_w + ox) * ch, px, ch);
    }
  return MFR_OK;
}

// ============================================================================================ PNG
// Gray 8- / 16-bit PNGs (the depth maps of lib/datasets/utils.py:77-81): a host chunk parser validates each file and
// builds its descriptor; one staging copy carries descriptors, the IDAT chunk table and each file's zlib stream (its
// IDAT payloads packed back to back); three kernels follow: CRC-32 of every IDAT (one CTA per file, long chunks split
// into pieces joined with crc_shift), inflate (one warp per file: lane 0 decodes from shared-memory tables into a 64 KB
// shared-memory window, two literals per lookup where both codes fit the root table, the warp copies long matches and
// stored runs, builds the tables and flushes the window to the filtered stream), unfilter + Adler-32 + output
// conversion (one CTA per file, rows in order).
namespace {

using png::Inflate;
using png::Layout;

constexpr uint32_t kPngPiece = 4096;       // CRC piece: long IDATs are split so that no thread walks a whole file
constexpr uint32_t kWinBytes = 1u << 16;   // inflate window ring: 32 KB of history + up to 32 KB pending flush
constexpr uint32_t kWarpMatch = 32;        // matches at least this long are copied by the whole warp
constexpr int kMaxSyms = 288 + 32;
__constant__ png::CrcTables c_crc = png::make_crc_tables();
constexpr png::CrcTables kCrcHost = png::make_crc_tables();

struct PngDesc {
  int width, height, depth, status, wbits, out_kind;
  uint32_t rowbytes, total;   // filtered stream: (1 + rowbytes) * height bytes
  uint32_t zlen;              // zlib stream bytes (header, deflate data, Adler-32 trailer)
  uint32_t adler;             // the trailer's value
  uint32_t nchunks, npieces;
  long long data;             // zlib stream: offset into the staged bytes
  long long chunk0, piece0;   // first IDAT entry / first CRC piece of the batch tables
  long long scratch;          // filtered stream: offset into the decoder's scratch (16-byte aligned)
  void* dst;
};

struct PngChunk {             // one IDAT: payload range in the file's zlib stream, stored CRC, first CRC piece
  uint32_t off, len, crc, piece0;
};

struct PngParsed {
  PngDesc d;
  std::vector<uint32_t> pos, len, crc;   // per IDAT: payload offset in the file, length, stored CRC
};

uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }

uint32_t crc_bytes(uint32_t reg, const uint8_t* p, uint32_t n) { return png::crc_update(kCrcHost.byte, reg, p, n); }
uint32_t crc_idat_state() { return crc_bytes(0xFFFFFFFFu, reinterpret_cast<const uint8_t*>("IDAT"), 4); }

// Parses and validates one file. MFR_OK: `out` describes a file the kernels decode; MFR_ERR_UNSUPPORTED: a valid file
// outside the supported set (colour types other than 0, bit depths 1 / 2 / 4, Adam7, chunks that change
// IMREAD_UNCHANGED's output or that this parser does not know, images beyond OpenCV's size limits); MFR_ERR_ARG:
// malformed structure (signature, chunk lengths, IHDR fields, chunk order, a missing IEND, the zlib header, the CRC of
// IHDR or IEND).
int parse_png(const uint8_t* data, size_t len, PngParsed& out) {
  static const uint8_t kSig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
  PngDesc& d = out.d;
  memset(&d, 0, sizeof(d));
  out.pos.clear(); out.len.clear(); out.crc.clear();
  if (!data || len < 8 + 25 || len > 0xFFFFFFFFull || memcmp(data, kSig, 8) != 0) return MFR_ERR_ARG;
  size_t p = 8;
  bool ihdr = false, iend = false, idat_done = false;
  int unsupported = 0;
  uint64_t zlen = 0;
  while (!iend) {
    if (p + 12 > len) return MFR_ERR_ARG;                  // truncated, or no IEND
    const uint32_t n = be32(data + p);
    const uint8_t* type = data + p + 4;
    if (n > 0x7FFFFFFFu || p + 12 + n > len) return MFR_ERR_ARG;
    for (int i = 0; i < 4; ++i)
      if (!((type[i] >= 'A' && type[i] <= 'Z') || (type[i] >= 'a' && type[i] <= 'z'))) return MFR_ERR_ARG;
    const uint8_t* body = data + p + 8;
    const uint32_t stored = be32(body + n);
    const bool is_idat = memcmp(type, "IDAT", 4) == 0;
    if (!ihdr && memcmp(type, "IHDR", 4) != 0) return MFR_ERR_ARG;   // IHDR comes first
    if (memcmp(type, "IHDR", 4) == 0) {
      if (ihdr || n != 13 || ~crc_bytes(0xFFFFFFFFu, type, 4 + n) != stored) return MFR_ERR_ARG;
      ihdr = true;
      const uint32_t w = be32(body), h = be32(body + 4);
      const int depth = body[8], color = body[9], comp = body[10], filter = body[11], interlace = body[12];
      if (w == 0 || h == 0 || w > 1000000u || h > 1000000u || comp != 0 || filter != 0 || interlace > 1) return MFR_ERR_ARG;
      const bool depth_ok = (color == 0 && (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)) ||
                            (color == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                            ((color == 2 || color == 4 || color == 6) && (depth == 8 || depth == 16));
      if (!depth_ok) return MFR_ERR_ARG;
      if (color != 0 || (depth != 8 && depth != 16) || interlace) unsupported = 1;
      // OpenCV's decoder refuses images over 2^30 pixels or 2^20 per side; those stay with it
      if (static_cast<uint64_t>(w) * h > (1ull << 30) || w > (1u << 20) || h > (1u << 20)) unsupported = 1;
      d.width = static_cast<int>(w); d.height = static_cast<int>(h); d.depth = depth;
    } else if (is_idat) {
      if (idat_done) return MFR_ERR_ARG;                   // IDATs must be consecutive
      out.pos.push_back(static_cast<uint32_t>(p + 8));
      out.len.push_back(n);
      out.crc.push_back(stored);
      zlen += n;
    } else {
      if (!out.pos.empty()) idat_done = true;
      if (memcmp(type, "IEND", 4) == 0) {
        if (n != 0 || out.pos.empty() || ~crc_bytes(0xFFFFFFFFu, type, 4) != stored) return MFR_ERR_ARG;
        iend = true;
      } else if (memcmp(type, "tEXt", 4) && memcmp(type, "zTXt", 4) && memcmp(type, "iTXt", 4) && memcmp(type, "tIME", 4) &&
                 memcmp(type, "pHYs", 4)) {
        unsupported = 1;                                   // PLTE, tRNS, sBIT, gAMA, iCCP, eXIf, acTL, unknown, ...
      }
    }
    p += 12 + n;
  }
  if (unsupported) return MFR_ERR_UNSUPPORTED;
  // zlib header and trailer, read across the IDAT boundaries
  if (zlen < 7 || zlen > 0xFFFFFFFFull) return MFR_ERR_ARG;
  auto zbyte = [&](uint64_t k) -> uint32_t {
    for (size_t c = 0; c < out.pos.size(); ++c) {
      if (k < out.len[c]) return data[out.pos[c] + k];
      k -= out.len[c];
    }
    return 0;
  };
  const uint32_t cmf = zbyte(0), flg = zbyte(1);
  if ((cmf & 15) != 8 || (cmf >> 4) > 7 || (cmf * 256 + flg) % 31 != 0 || (flg & 0x20)) return MFR_ERR_ARG;
  d.wbits = static_cast<int>(cmf >> 4) + 8;
  d.adler = (zbyte(zlen - 4) << 24) | (zbyte(zlen - 3) << 16) | (zbyte(zlen - 2) << 8) | zbyte(zlen - 1);
  d.zlen = static_cast<uint32_t>(zlen);
  d.rowbytes = static_cast<uint32_t>(d.width) * (d.depth / 8);
  const uint64_t total = (1ull + d.rowbytes) * static_cast<uint64_t>(d.height);
  if (total > 0xFFFF0000ull) return MFR_ERR_UNSUPPORTED;
  d.total = static_cast<uint32_t>(total);
  d.nchunks = static_cast<uint32_t>(out.pos.size());
  d.npieces = 0;
  for (uint32_t l : out.len) d.npieces += (l + kPngPiece - 1) / kPngPiece;
  d.status = MFR_OK;
  return MFR_OK;
}

// ------------------------------------------------------------------------------------------ kernels
// CRC-32 of every IDAT of file blockIdx.x: per piece crc_update (the first piece of a chunk starting from the register
// after "IDAT"), then per chunk its pieces joined in order.
__global__ void __launch_bounds__(256) png_crc_kernel(const PngDesc* __restrict__ descs, const PngChunk* __restrict__ chunks,
                                                      const uint32_t* __restrict__ piece_chunk, const uint8_t* __restrict__ data,
                                                      uint32_t* __restrict__ piece_crc, uint32_t idat_state,
                                                      int* __restrict__ status) {
  __shared__ uint32_t table[256];
  const PngDesc& d = descs[blockIdx.x];
  if (d.status != MFR_OK) return;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) table[i] = c_crc.byte[i];
  __syncthreads();
  const uint8_t* z = data + d.data;
  for (uint32_t q = threadIdx.x; q < d.npieces; q += blockDim.x) {
    const long long pi = d.piece0 + q;
    const PngChunk c = chunks[piece_chunk[pi]];
    const uint32_t k = static_cast<uint32_t>(pi - c.piece0), off = k * kPngPiece;
    const uint32_t n = min(kPngPiece, c.len - off);
    piece_crc[pi] = png::crc_update(table, k ? 0u : idat_state, z + c.off + off, n);
  }
  __syncthreads();
  for (uint32_t ci = threadIdx.x; ci < d.nchunks; ci += blockDim.x) {
    const PngChunk c = chunks[d.chunk0 + ci];
    const uint32_t np = (c.len + kPngPiece - 1) / kPngPiece;
    uint32_t reg = np ? piece_crc[c.piece0] : idat_state;
    for (uint32_t k = 1; k < np; ++k) reg = png::crc_shift(c_crc.x2n, reg, min(kPngPiece, c.len - k * kPngPiece)) ^ piece_crc[c.piece0 + k];
    if (~reg != c.crc) status[blockIdx.x] = MFR_ERR_ARG;
  }
}

// One warp per file: the filtered stream (1 + rowbytes) x height into the scratch.
__global__ void __launch_bounds__(32) png_inflate_kernel(const PngDesc* __restrict__ descs, const uint8_t* __restrict__ data,
                                                         uint8_t* __restrict__ scratch, int* __restrict__ status) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ Layout lay[2];
  __shared__ uint32_t regions[2][png::kMaxRegions];
  uint32_t* lit = reinterpret_cast<uint32_t*>(smem);
  uint32_t* dist = lit + png::kTableCap;
  uint32_t* pair = dist + png::kTableCap;
  uint8_t* win = reinterpret_cast<uint8_t*>(pair + (1 << png::kRootBits));
  uint16_t* codes = reinterpret_cast<uint16_t*>(win + kWinBytes);
  uint8_t* lens = reinterpret_cast<uint8_t*>(codes + kMaxSyms);
  const PngDesc& d = descs[blockIdx.x];
  if (d.status != MFR_OK) return;
  const int lane = threadIdx.x;
  const uint8_t* z = data + d.data + 2;                   // deflate data after the zlib header (16-byte aligned)
  uint8_t* out = scratch + d.scratch;
  if (lane < 2) lay[lane].region = regions[lane];
  __syncwarp();
  Inflate s;
  png::inflate_init(s, reinterpret_cast<const uint32_t*>(z), d.zlen - 6, win, kWinBytes - 1, kWinBytes / 2, d.total, d.wbits);
  for (;;) {
    int cmd = 0;
    if (lane == 0) cmd = png::inflate_run(s, lit, pair, dist, lens, codes, lay, kWarpMatch);
    cmd = __shfl_sync(0xFFFFFFFFu, cmd, 0);
    const uint32_t o = __shfl_sync(0xFFFFFFFFu, s.cmd_out, 0), n = __shfl_sync(0xFFFFFFFFu, s.cmd_len, 0);
    const uint32_t dd = __shfl_sync(0xFFFFFFFFu, s.cmd_dist, 0), cur = __shfl_sync(0xFFFFFFFFu, s.out, 0);
    const uint32_t fl = __shfl_sync(0xFFFFFFFFu, s.flushed, 0);
    __syncwarp();
    if (cmd == png::kCmdMatch) {
      if (dd >= 32) {
        for (uint32_t b = 0; b < n; b += 32) {            // each 32-byte step reads bytes the previous steps wrote
          const uint32_t i = b + lane;
          if (i < n) win[(o + i) & (kWinBytes - 1)] = win[(o + i - dd) & (kWinBytes - 1)];
          __syncwarp();
        }
      } else {                                            // short period: read the pattern before the match
        for (uint32_t i = lane; i < n; i += 32) win[(o + i) & (kWinBytes - 1)] = win[(o - dd + i % dd) & (kWinBytes - 1)];
      }
    } else if (cmd == png::kCmdStored) {
      for (uint32_t i = lane; i < n; i += 32) win[(o + i) & (kWinBytes - 1)] = z[dd + i];
    } else if (cmd == png::kCmdBuild) {
      const int nl = __shfl_sync(0xFFFFFFFFu, s.nlen, 0), nd = __shfl_sync(0xFFFFFFFFu, s.ndist, 0);
      png::huff_fill_invalid(lit, lane, 32);
      png::huff_fill_invalid(dist, lane, 32);
      __syncwarp();
      png::huff_fill(lens, codes, nl, 0, lay[0], lit, lane, 32);
      png::huff_fill(lens + nl, codes + nl, nd, 1, lay[1], dist, lane, 32);
      __syncwarp();
      png::huff_fill_pairs(lit, pair, lane, 32);
    } else if (cmd == png::kCmdFlush || cmd == png::kCmdDone) {
      for (uint32_t i = fl + lane; i < cur; i += 32) out[i] = win[i & (kWinBytes - 1)];
      if (lane == 0) s.flushed = cur;
    } else {
      if (lane == 0) status[blockIdx.x] = MFR_ERR_ARG;
    }
    __syncwarp();
    if (cmd == png::kCmdDone || cmd == png::kCmdError) break;
  }
}

constexpr int kUnfilterThreads = 256;

// exclusive scan over the CTA of per-thread packed byte-lane sums (lane c in bits 16c..16c+7, mod 256)
__device__ uint32_t block_scan_bytes(uint32_t v, uint32_t* warp_tot) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t inc = v;
  for (int k = 1; k < 32; k <<= 1) {
    const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, inc, k);
    if (lane >= k) inc = (inc + u) & 0x00FF00FFu;
  }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  uint32_t pre = 0;
  for (int i = 0; i < w; ++i) pre = (pre + warp_tot[i]) & 0x00FF00FFu;
  __syncthreads();
  return (pre + inc - v + 0x01000100u) & 0x00FF00FFu;     // + 256 per lane keeps inc - v from borrowing across lanes
}

// One CTA per file: Adler-32 of the filtered stream against the trailer, then per row: unfilter in place (None / Up
// elementwise, Sub as a scan per byte lane, Average / Paeth serially per byte lane), convert into dst.
__global__ void __launch_bounds__(kUnfilterThreads) png_unfilter_kernel(const PngDesc* __restrict__ descs, uint8_t* __restrict__ scratch,
                                                                       int* __restrict__ status) {
  __shared__ unsigned long long red[2][kUnfilterThreads / 32];
  __shared__ uint32_t warp_tot[kUnfilterThreads / 32];
  const PngDesc& d = descs[blockIdx.x];
  if (d.status != MFR_OK || status[blockIdx.x] != MFR_OK) return;
  uint8_t* f = scratch + d.scratch;
  const int tid = threadIdx.x, T = blockDim.x;
  // Adler-32: S1 = sum of bytes, S2 = sum of position * byte, 16 bytes per step (the scratch is 16-byte aligned and padded)
  unsigned long long s1 = 0, s2 = 0;
  for (uint32_t v = tid; static_cast<uint64_t>(v) * 16 < d.total; v += T) {
    const uint32_t base = v * 16, jm = base % png::kAdlerMod;
    const uint4 q = reinterpret_cast<const uint4*>(f)[v];
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int b = 0; b < 16; ++b) {
      const uint32_t x = base + b < d.total ? (w[b >> 2] >> (8 * (b & 3))) & 0xFF : 0;
      s1 += x;
      s2 += static_cast<unsigned long long>(jm + b) * x;
    }
  }
  for (int k = 16; k; k >>= 1) {
    s1 += __shfl_down_sync(0xFFFFFFFFu, s1, k);
    s2 += __shfl_down_sync(0xFFFFFFFFu, s2, k);
  }
  if ((tid & 31) == 0) { red[0][tid >> 5] = s1; red[1][tid >> 5] = s2; }
  __syncthreads();
  s1 = s2 = 0;
  for (int i = 0; i < T / 32; ++i) { s1 += red[0][i]; s2 += red[1][i]; }
  if (png::adler_from_sums(d.total, s1, s2) != d.adler) {
    if (tid == 0) status[blockIdx.x] = MFR_ERR_ARG;
    return;
  }
  const int bpp = d.depth / 8;
  const uint32_t rb = d.rowbytes, ne = rb / bpp, span = (ne + T - 1) / T;
  for (int r = 0; r < d.height; ++r) {
    uint8_t* row = f + static_cast<uint64_t>(r) * (rb + 1);
    uint8_t* cur = row + 1;
    const uint8_t* prev = r ? row - rb : nullptr;
    const int ft = row[0];
    if (ft > 4) {
      if (tid == 0) status[blockIdx.x] = MFR_ERR_ARG;
      return;
    }
    if (ft == 2 && prev) {
      for (uint32_t i = tid; i < rb; i += T) cur[i] = static_cast<uint8_t>(cur[i] + prev[i]);
    } else if (ft == 1) {
      const uint32_t e0 = min(ne, tid * span), e1 = min(ne, e0 + span);
      uint32_t acc = 0;
      for (uint32_t e = e0; e < e1; ++e)
        for (int c = 0; c < bpp; ++c) acc = (acc + (static_cast<uint32_t>(cur[e * bpp + c]) << (16 * c))) & 0x00FF00FFu;
      uint32_t run = block_scan_bytes(acc, warp_tot);
      for (uint32_t e = e0; e < e1; ++e)
        for (int c = 0; c < bpp; ++c) {
          const uint32_t v = (cur[e * bpp + c] + (run >> (16 * c))) & 0xFF;
          cur[e * bpp + c] = static_cast<uint8_t>(v);
          run = (run & ~(0xFFu << (16 * c))) | (v << (16 * c));
        }
    } else if (ft >= 3 && tid < bpp) {
      int a = 0, c = 0;
      for (uint32_t i0 = tid; i0 < rb; i0 += 8 * bpp) {
        int x[8], u[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const uint32_t i = i0 + k * bpp;
          x[k] = i < rb ? cur[i] : 0;
          u[k] = (prev && i < rb) ? prev[i] : 0;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int v = (x[k] + (ft == 3 ? (a + u[k]) >> 1 : png::paeth(a, u[k], c))) & 0xFF;
          c = u[k];
          a = v;
          x[k] = v;
        }
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (i0 + k * bpp < rb) cur[i0 + k * bpp] = static_cast<uint8_t>(x[k]);
      }
    }
    __syncthreads();
    for (int x = tid; x < d.width; x += T) png::store_sample(cur, x, d.depth, d.out_kind, d.dst, static_cast<uint64_t>(r) * d.width + x);
  }
}

size_t png_smem_bytes() { return (2 * png::kTableCap + (1 << png::kRootBits)) * 4 + kWinBytes + kMaxSyms * 2 + kMaxSyms; }

}  // namespace

// ------------------------------------------------------------------------------------------ PNG decoder
struct PngDecoder {
  int max_images = 0;
  long long max_bytes = 0, scratch_cap = 0, chunk_cap = 0, piece_cap = 0;
  Staging stage;
  uint8_t* scratch = nullptr;
  uint32_t* piece_crc = nullptr;
  cudaEvent_t ev[4] = {};   // around the last batch's kernels: CRC, inflate, unfilter
  std::vector<PngParsed> parsed;
};

void png_decoder_destroy(PngDecoder* dec) {
  if (!dec) return;
  staging_destroy(dec->stage);
  for (cudaEvent_t e : dec->ev)
    if (e) cudaEventDestroy(e);
  cudaFree(dec->scratch);
  cudaFree(dec->piece_crc);
  delete dec;
}

int png_decoder_create(int max_images, long long max_bytes, long long max_pixels, PngDecoder** out) {
  if (!out || max_images < 1 || max_images > 65535 || max_bytes < 1 || max_pixels < 1) return MFR_ERR_ARG;
  *out = nullptr;
  PngDecoder* dec = new PngDecoder();
  dec->max_images = max_images;
  dec->max_bytes = max_bytes;
  dec->scratch_cap = 3 * max_pixels + 16ll * max_images + 16;     // (1 + 2w) h <= 3 w h, 16-byte aligned per file
  dec->chunk_cap = max_bytes / 12 + max_images;                    // a chunk takes 12 bytes of its file at least
  dec->piece_cap = dec->chunk_cap + max_bytes / kPngPiece + max_images;
  const size_t stage_bytes = align_up(static_cast<size_t>(max_images) * sizeof(PngDesc), 256) + align_up(4ull * max_images, 256) +
                             align_up(sizeof(PngChunk) * dec->chunk_cap, 256) + align_up(4ull * dec->piece_cap, 256) +
                             static_cast<size_t>(max_bytes);
  const bool ok = staging_create(dec->stage, stage_bytes) && cudaMalloc(&dec->scratch, dec->scratch_cap) == cudaSuccess &&
                  cudaMalloc(&dec->piece_crc, 4ull * dec->piece_cap) == cudaSuccess &&
                  cudaEventCreate(&dec->ev[0]) == cudaSuccess && cudaEventCreate(&dec->ev[1]) == cudaSuccess &&
                  cudaEventCreate(&dec->ev[2]) == cudaSuccess && cudaEventCreate(&dec->ev[3]) == cudaSuccess;
  if (!ok) {
    png_decoder_destroy(dec);
    return MFR_ERR_CUDA;
  }
  dec->parsed.resize(max_images);
  *out = dec;
  return MFR_OK;
}

int png_info(const unsigned char* data, size_t length, int* width, int* height, int* bit_depth) {
  PngParsed p;
  const int rc = parse_png(data, length, p);
  if (rc != MFR_OK) return rc;
  *width = p.d.width; *height = p.d.height; *bit_depth = p.d.depth;
  return MFR_OK;
}

void png_batch_info(const unsigned char* const* data, const long long* lengths, int n, int* width, int* height, int* bit_depth,
                    int* status) {
  PngParsed p;
  for (int i = 0; i < n; ++i) {
    status[i] = (data[i] && lengths[i] > 0) ? parse_png(data[i], static_cast<size_t>(lengths[i]), p) : MFR_ERR_ARG;
    const bool ok = status[i] == MFR_OK;
    width[i] = ok ? p.d.width : 0;
    height[i] = ok ? p.d.height : 0;
    bit_depth[i] = ok ? p.d.depth : 0;
  }
}

int png_decode_batch(PngDecoder* dec, const unsigned char* const* data, const long long* lengths, int n, int out_kind,
                     void* const* dst, int* status, cudaStream_t st) {
  if (!dec || n < 0 || n > dec->max_images || (out_kind != 0 && out_kind != 1) ||
      (n > 0 && (!data || !lengths || !dst || !status)))
    return MFR_ERR_ARG;
  if (n == 0) return MFR_OK;
  long long bytes = 0, scratch = 0, chunks = 0, pieces = 0;
  for (int i = 0; i < n; ++i) {
    PngParsed& p = dec->parsed[i];
    int rc = (data[i] && lengths[i] > 0) ? parse_png(data[i], static_cast<size_t>(lengths[i]), p) : MFR_ERR_ARG;
    if (rc == MFR_OK && !dst[i]) rc = MFR_ERR_ARG;
    if (rc != MFR_OK) { memset(&p.d, 0, sizeof(PngDesc)); p.d.status = rc; p.pos.clear(); continue; }
    PngDesc& d = p.d;
    d.out_kind = out_kind;
    d.dst = dst[i];
    d.data = static_cast<long long>(align_up(static_cast<size_t>(bytes) + 2, 16)) - 2;   // deflate data 16-byte aligned
    bytes = d.data;
    d.chunk0 = chunks;
    d.piece0 = pieces;
    d.scratch = scratch;
    bytes += d.zlen;
    chunks += d.nchunks;
    pieces += d.npieces;
    scratch += static_cast<long long>(align_up(d.total, 16));
  }
  if (bytes > dec->max_bytes || scratch + 16 > dec->scratch_cap || chunks > dec->chunk_cap || pieces > dec->piece_cap)
    return MFR_ERR_ARG;                                     // over capacity
  // staging layout: descriptors | initial statuses | IDAT table | piece -> IDAT | zlib streams
  const size_t off_status = align_up(static_cast<size_t>(n) * sizeof(PngDesc), 256);
  const size_t off_chunks = off_status + align_up(4ull * n, 256);
  const size_t off_pieces = off_chunks + align_up(sizeof(PngChunk) * chunks, 256);
  const size_t off_data = off_pieces + align_up(4ull * pieces, 256);
  const size_t total = off_data + static_cast<size_t>(bytes);
  int rc = staging_acquire(dec->stage);
  if (rc != MFR_OK) return rc;
  unsigned char* h = dec->stage.h;
  PngDesc* hd = reinterpret_cast<PngDesc*>(h);
  int* hs = reinterpret_cast<int*>(h + off_status);
  PngChunk* hc = reinterpret_cast<PngChunk*>(h + off_chunks);
  uint32_t* hp = reinterpret_cast<uint32_t*>(h + off_pieces);
  for (int i = 0; i < n; ++i) {
    const PngParsed& p = dec->parsed[i];
    hd[i] = p.d;
    hs[i] = p.d.status;
    if (p.d.status != MFR_OK) continue;
    uint32_t off = 0;
    long long piece = p.d.piece0;
    for (size_t c = 0; c < p.pos.size(); ++c) {
      const long long ci = p.d.chunk0 + static_cast<long long>(c);
      hc[ci] = PngChunk{off, p.len[c], p.crc[c], static_cast<uint32_t>(piece)};
      for (uint32_t k = 0; k < (p.len[c] + kPngPiece - 1) / kPngPiece; ++k) hp[piece++] = static_cast<uint32_t>(ci);
      memcpy(h + off_data + p.d.data + off, data[i] + p.pos[c], p.len[c]);
      off += p.len[c];
    }
  }
  rc = staging_upload(dec->stage, total, st);
  if (rc != MFR_OK) return rc;
  const unsigned char* ds = dec->stage.d;
  const PngDesc* dd = reinterpret_cast<const PngDesc*>(ds);
  MFR_CUDA_CHECK(cudaMemcpyAsync(status, ds + off_status, 4ull * n, cudaMemcpyDeviceToDevice, st));
  if (bytes > 0) {
    static bool attr_seen[64] = {};   // the shared-memory opt-in is per device
    if (first_call_on_device(attr_seen))
      MFR_CUDA_CHECK(cudaFuncSetAttribute(png_inflate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          static_cast<int>(png_smem_bytes())));
    MFR_CUDA_CHECK(cudaEventRecord(dec->ev[0], st));
    png_crc_kernel<<<n, 256, 0, st>>>(dd, reinterpret_cast<const PngChunk*>(ds + off_chunks),
                                      reinterpret_cast<const uint32_t*>(ds + off_pieces), ds + off_data, dec->piece_crc,
                                      crc_idat_state(), status);
    MFR_CUDA_CHECK(cudaEventRecord(dec->ev[1], st));
    png_inflate_kernel<<<n, 32, png_smem_bytes(), st>>>(dd, ds + off_data, dec->scratch, status);
    MFR_CUDA_CHECK(cudaEventRecord(dec->ev[2], st));
    png_unfilter_kernel<<<n, kUnfilterThreads, 0, st>>>(dd, dec->scratch, status);
    MFR_CUDA_CHECK(cudaEventRecord(dec->ev[3], st));
    MFR_CUDA_CHECK(cudaGetLastError());
  }
  return staging_release(dec->stage, st);
}

// Milliseconds of the CRC, inflate and unfilter kernels of the decoder's last batch that launched them (waits for it).
int png_decoder_kernel_ms(PngDecoder* dec, float* ms) {
  MFR_CUDA_CHECK(cudaEventSynchronize(dec->ev[3]));
  for (int k = 0; k < 3; ++k) MFR_CUDA_CHECK(cudaEventElapsedTime(ms + k, dec->ev[k], dec->ev[k + 1]));
  return MFR_OK;
}

// The same arithmetic serially on the CPU (test hook): dst [height][width] of uint8 / uint16 (kind 0) or float32
// (kind 1), host memory.
int png_host_decode(const unsigned char* data, size_t length, int out_kind, void* dst, int width, int height) {
  PngParsed p;
  const int rc = parse_png(data, length, p);
  if (rc != MFR_OK) return rc;
  const PngDesc& d = p.d;
  if (d.width != width || d.height != height || (out_kind != 0 && out_kind != 1)) return MFR_ERR_ARG;
  std::vector<uint8_t> z;
  z.reserve(d.zlen);
  for (size_t c = 0; c < p.pos.size(); ++c) {
    const uint8_t* body = data + p.pos[c];
    if (~crc_bytes(crc_idat_state(), body, p.len[c]) != p.crc[c]) return MFR_ERR_ARG;
    z.insert(z.end(), body, body + p.len[c]);
  }
  std::vector<uint32_t> words((d.zlen - 6 + 3) / 4 + 1, 0);  // the deflate data, 4-byte aligned as on the device
  memcpy(words.data(), z.data() + 2, d.zlen - 6);
  std::vector<uint8_t> f(d.total);
  std::vector<uint32_t> lit(png::kTableCap), dist(png::kTableCap), pair(1 << png::kRootBits);
  uint8_t lens[kMaxSyms];
  uint16_t codes[kMaxSyms];
  uint32_t regions[2][png::kMaxRegions];
  Layout lay[2];
  lay[0].region = regions[0];
  lay[1].region = regions[1];
  Inflate s;
  png::inflate_init(s, words.data(), d.zlen - 6, f.data(), 0xFFFFFFFFu, 0xFFFFFFFFu, d.total, d.wbits);
  for (int cmd = 0; cmd != png::kCmdDone;) {
    cmd = png::inflate_run(s, lit.data(), pair.data(), dist.data(), lens, codes, lay, 0xFFFFFFFFu);
    if (cmd == png::kCmdError) return MFR_ERR_ARG;
    if (cmd == png::kCmdStored) memcpy(f.data() + s.cmd_out, reinterpret_cast<const uint8_t*>(words.data()) + s.cmd_dist, s.cmd_len);
    if (cmd == png::kCmdBuild) {
      png::huff_fill_invalid(lit.data(), 0, 1);
      png::huff_fill_invalid(dist.data(), 0, 1);
      png::huff_fill(lens, codes, s.nlen, 0, lay[0], lit.data(), 0, 1);
      png::huff_fill(lens + s.nlen, codes + s.nlen, s.ndist, 1, lay[1], dist.data(), 0, 1);
      png::huff_fill_pairs(lit.data(), pair.data(), 0, 1);
    }
  }
  uint64_t s1 = 0, s2 = 0;
  for (uint32_t j = 0; j < d.total; ++j) { s1 += f[j]; s2 += static_cast<uint64_t>(j % png::kAdlerMod) * f[j]; }
  if (png::adler_from_sums(d.total, s1, s2) != d.adler) return MFR_ERR_ARG;
  const uint32_t rb = d.rowbytes;
  for (int r = 0; r < d.height; ++r) {
    uint8_t* row = f.data() + static_cast<size_t>(r) * (rb + 1);
    if (png::unfilter_row(row[0], row + 1, r ? row - rb : nullptr, rb, d.depth / 8)) return MFR_ERR_ARG;
    for (int x = 0; x < d.width; ++x) png::store_sample(row + 1, x, d.depth, out_kind, dst, static_cast<uint64_t>(r) * d.width + x);
  }
  return MFR_OK;
}

}  // namespace mfr
