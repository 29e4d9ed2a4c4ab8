// Input path of the matchers on the GPU (SURVEY §8(f) rank 1): JPEG decode (the arithmetic of cv2.imread, jpeg.cuh) +
// the resize / normalise step of the reference's loaders
//   read_image      etc/feature_matching_baselines/SuperGlue/models/utils.py:263-285   gray, cv2.resize, / 255
//   read_color_image lib/datasets/utils.py:58-75                                        RGB uint8 cv2.resize, / 255, CHW
// cv2.resize(INTER_LINEAR) is restated for both of its code paths: float32 images (bilinear weights in fp32, horizontal
// pass first) and uint8 images (11-bit fixed-point weights, OpenCV's two-stage rounding), so that the resized pixels are
// the ones the reference feeds its networks. 16-bit depth PNGs (read_depth_image) stay on the host: inflate is not GPU work.
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

// ------------------------------------------------------------------------------------------ decoder
struct JpegDecoder {
  int max_images = 0;
  long long max_bytes = 0, sample_cap = 0, unit_cap = 0;
  size_t stage_bytes = 0;
  unsigned char* h_stage = nullptr;   // pinned
  unsigned char* d_stage = nullptr;
  int16_t* coef = nullptr;
  uint8_t* planes = nullptr;
  cudaEvent_t copied = nullptr, done = nullptr;
  std::vector<Parsed> parsed;
};

void jpeg_decoder_destroy(JpegDecoder* dec) {
  if (!dec) return;
  if (dec->done) cudaEventSynchronize(dec->done);
  if (dec->copied) cudaEventDestroy(dec->copied);
  if (dec->done) cudaEventDestroy(dec->done);
  if (dec->h_stage) cudaFreeHost(dec->h_stage);
  cudaFree(dec->d_stage);
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
  dec->stage_bytes = align_up(static_cast<size_t>(max_images) * sizeof(Desc), 256) + align_up(4ull * max_images, 256) +
                     align_up(4ull * dec->unit_cap, 256) + static_cast<size_t>(max_bytes);
  bool ok = cudaHostAlloc(&dec->h_stage, dec->stage_bytes, cudaHostAllocDefault) == cudaSuccess &&
            cudaMalloc(&dec->d_stage, dec->stage_bytes) == cudaSuccess &&
            cudaMalloc(&dec->coef, 2 * dec->sample_cap) == cudaSuccess &&
            cudaMalloc(&dec->planes, dec->sample_cap) == cudaSuccess &&
            cudaEventCreateWithFlags(&dec->copied, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventCreateWithFlags(&dec->done, cudaEventDisableTiming) == cudaSuccess;
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
  MFR_CUDA_CHECK(cudaEventSynchronize(dec->copied));        // the previous call's staging has reached the device
  unsigned char* h = dec->h_stage;
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
  MFR_CUDA_CHECK(cudaStreamWaitEvent(st, dec->done, 0));     // the previous call's kernels are done with the buffers
  MFR_CUDA_CHECK(cudaMemcpyAsync(dec->d_stage, h, total, cudaMemcpyHostToDevice, st));
  MFR_CUDA_CHECK(cudaEventRecord(dec->copied, st));
  const Desc* dd = reinterpret_cast<const Desc*>(dec->d_stage);
  MFR_CUDA_CHECK(cudaMemcpyAsync(status, dec->d_stage + off_status, 4ull * n, cudaMemcpyDeviceToDevice, st));
  if (samples > 0) {
    MFR_CUDA_CHECK(cudaMemsetAsync(dec->coef, 0, 2ull * samples, st));
    jpeg_entropy_kernel<<<dim3((max_units + 63) / 64, n), 64, 0, st>>>(
        dd, reinterpret_cast<const uint32_t*>(dec->d_stage + off_units), dec->d_stage + off_data, dec->coef, status);
    jpeg_idct_kernel<<<dim3((max_blocks + 127) / 128, n), 128, 0, st>>>(dd, dec->coef, dec->planes);
    jpeg_pixel_kernel<<<dim3(static_cast<unsigned>((max_px + 255) / 256), n), 256, 0, st>>>(dd, dec->planes);
    MFR_CUDA_CHECK(cudaGetLastError());
  }
  MFR_CUDA_CHECK(cudaEventRecord(dec->done, st));
  return MFR_OK;
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

}  // namespace mfr
