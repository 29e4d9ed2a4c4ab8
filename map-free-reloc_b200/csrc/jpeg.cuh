// Baseline JPEG decode as libjpeg(-turbo) computes it, the arithmetic of cv2.imread (ITU T.81 + libjpeg's documented
// decompression defaults: JDCT_ISLOW, fancy upsampling, 16-bit fixed-point YCbCr -> RGB). Every per-unit, per-block and
// per-pixel step is an MFR_HD function, so the CUDA kernels of image_io.cu and the serial CPU hook mfr_host_jpeg_decode
// run one copy of it. The host parser (image_io.cu) fills a jpeg::Desc per image; it has validated everything the loops
// below rely on (table completeness, block counts, byte ranges), so they only bound-check the entropy-coded data.
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define MFR_HD __host__ __device__ __forceinline__
#else
#define MFR_HD inline
#endif

namespace mfr {
namespace jpeg {

constexpr int kLutBits = 9;       // codes of <= 9 bits resolve in one lookup; longer ones walk maxcode (T.81 F.2.2.3)
constexpr int kMaxTables = 6;     // distinct (DC, AC) tables one scan of <= 3 components can reference

struct Huff {
  uint16_t lut[1 << kLutBits];    // (length << 8) | symbol for codes of <= kLutBits bits, 0: longer code
  int32_t maxcode[18];            // largest code of each length 1..16, -1 if none; [17] = sentinel
  int32_t valoff[17];             // vals index of a code of length l = code + valoff[l]
  uint8_t vals[256];
};

struct Comp {
  int h, v;                       // sampling factors in the scan's MCU (1 x 1 for a one-component scan)
  int bw, bh;                     // blocks per row / column of the coefficient plane (whole MCUs)
  int dw, dh;                     // downsampled width / height (libjpeg's downsampled_width / height)
  int dc, ac;                     // indices into JpegDesc::tbl
  long long coef;                 // first coefficient of the plane in the decoder's int16 buffer
  long long plane;                // first sample of the plane in the decoder's uint8 buffer (stride bw * 8)
};

struct Desc {
  int width, height;              // as coded (SOF)
  int out_w, out_h;               // after the Exif orientation (5-8 swap them)
  int orient;                     // Exif Orientation 1-8
  int ncomp, hmax, vmax;
  int mcus_x, mcus_y, restart;    // restart: MCUs per restart interval, 0: none
  int n_units, n_blocks;          // decode units (one image, or one restart interval each); blocks of all planes
  int n_tbl;                      // Huffman tables in use (tbl[0 .. n_tbl))
  int rgb;
  int status;                     // MFR_OK, or why the host did not launch this image
  long long data;                 // entropy-coded bytes: offset into the staged byte array
  long long units;                // offset into the staged uint32 array: per unit its byte range (start, end) in data
  unsigned char* dst;
  Comp comp[3];
  int32_t qt[3][64];              // per component, natural order, as libjpeg's ISLOW multiplier table holds them (int16)
  Huff tbl[kMaxTables];
};

// natural order of the k-th zig-zag coefficient, padded with 16 entries of 63 so that a corrupt run (k up to 63 + 15)
// lands on 63 as libjpeg's table does; the kernels keep a shared-memory copy, the host hook this one
#define MFR_JPEG_NATURAL_ORDER                                                                                          \
  {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,         \
   6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,         \
   39, 46, 53, 60, 61, 54, 47, 55, 62, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63}
constexpr int kNaturalLen = 80;

// ------------------------------------------------------------------------------------------ entropy decode
// MSB-first bit reader over one unit's bytes [p, end): FF00 unstuffed; past the end (or at a marker) it shifts in zero
// bits and counts them, and consuming one of those is an error (libjpeg warns and decodes zeros; the caller then falls
// back to it).
struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  uint64_t acc;
  int nbits, fake;
  MFR_HD void fill() {
    while (nbits <= 56) {
      unsigned b = 0;
      if (p < end && fake == 0) {
        b = *p++;
        if (b == 0xFF) {
          if (p < end && *p == 0x00) ++p;
          else { b = 0; fake += 8; p = end; }
        }
      } else {
        fake += 8;
      }
      acc = (acc << 8) | b;
      nbits += 8;
    }
  }
  MFR_HD unsigned peek(int n) const { return static_cast<unsigned>(acc >> (nbits - n)) & ((1u << n) - 1u); }
  MFR_HD bool overrun() const { return nbits < fake; }
};

// one Huffman symbol (the reader holds >= 32 bits); -1: no code of <= 16 bits matches
MFR_HD int huff_decode(BitReader& br, const Huff& t) {
  const unsigned e = t.lut[br.peek(kLutBits)];
  if (e) { br.nbits -= e >> 8; return e & 0xFF; }
  const int code16 = static_cast<int>(br.peek(16));
  for (int l = kLutBits + 1; l <= 16; ++l) {
    const int c = code16 >> (16 - l);
    if (c <= t.maxcode[l]) { br.nbits -= l; return t.vals[c + t.valoff[l]]; }
  }
  return -1;
}

// s (1..15) magnitude bits -> signed value (T.81 F.2.2.1 EXTEND)
MFR_HD int receive_extend(BitReader& br, int s) {
  const int v = static_cast<int>(br.peek(s));
  br.nbits -= s;
  return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v;
}

// Decodes unit u (restart interval u, or the whole scan) into the zero-filled coefficient buffer: DC prediction from 0
// at the unit's start, int16 coefficients in natural order. Returns 0, or 1 on an invalid code / data overrun.
MFR_HD int decode_unit(const Desc& d, const Huff* tbl, const uint8_t* nat, const uint8_t* data, const uint32_t* units, int u,
                       int16_t* coef) {
  BitReader br{data + units[2 * u], data + units[2 * u + 1], 0, 0, 0};
  const int total = d.mcus_x * d.mcus_y;
  const int m0 = d.restart ? u * d.restart : 0;
  const int m1 = d.restart ? (m0 + d.restart < total ? m0 + d.restart : total) : total;
  int pred[3] = {0, 0, 0};
  for (int m = m0; m < m1; ++m) {
    const int mx = m % d.mcus_x, my = m / d.mcus_x;
    for (int c = 0; c < d.ncomp; ++c) {
      const Comp& cp = d.comp[c];
      const Huff& dc = tbl[cp.dc];
      const Huff& ac = tbl[cp.ac];
      for (int by = 0; by < cp.v; ++by)
        for (int bx = 0; bx < cp.h; ++bx) {
          int16_t* blk = coef + cp.coef + ((static_cast<long long>(my * cp.v + by) * cp.bw + mx * cp.h + bx) << 6);
          br.fill();
          const int s = huff_decode(br, dc);
          if (s < 0) return 1;
          if (s) pred[c] += receive_extend(br, s);
          blk[0] = static_cast<int16_t>(pred[c]);
          for (int k = 1; k < 64; ++k) {
            br.fill();
            const int rs = huff_decode(br, ac);
            if (rs < 0) return 1;
            const int r = rs >> 4, sz = rs & 15;
            if (sz) {
              k += r;
              blk[nat[k]] = static_cast<int16_t>(receive_extend(br, sz));
            } else {
              if (r != 15) break;
              k += 15;
            }
          }
        }
    }
    if (br.overrun()) return 1;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------ dequantise + ISLOW IDCT
// libjpeg's jpeg_idct_islow: Loeffler-Ligtenberg-Moschytz, CONST_BITS 13, PASS1_BITS 2, DESCALE = round half up by
// adding 2^(n-1) before the arithmetic shift; the output goes through the post-IDCT range-limit table, indexed by the
// low 10 bits of the result, so out-of-range values saturate within +-512 of the range and wrap beyond it.
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int32_t kF0298 = 2446, kF0390 = 3196, kF0541 = 4433, kF0765 = 6270, kF0899 = 7373, kF1175 = 9633,
                  kF1501 = 12299, kF1847 = 15137, kF1961 = 16069, kF2053 = 16819, kF2562 = 20995, kF3072 = 25172;

MFR_HD int64_t descale(int64_t x, int n) { return (x + (int64_t(1) << (n - 1))) >> n; }

// libjpeg's post-IDCT range limit of a centred sample x (masked to 10 bits, +128 level shift)
MFR_HD uint8_t idct_limit(int64_t x) {
  const int m = static_cast<int>(x & 1023);
  if (m < 128) return static_cast<uint8_t>(m + 128);
  if (m < 512) return 255;
  if (m < 896) return 0;
  return static_cast<uint8_t>(m - 896);
}

// the LLM butterfly on inputs i0..i7 (JLONG arithmetic, 64-bit as libjpeg's on LP64): out[0..7] before the descale
MFR_HD void idct_1d(int64_t i0, int64_t i1, int64_t i2, int64_t i3, int64_t i4, int64_t i5, int64_t i6, int64_t i7, int64_t* o) {
  int64_t z1 = (i2 + i6) * kF0541;
  const int64_t t2 = z1 + i6 * -kF1847, t3 = z1 + i2 * kF0765;
  const int64_t t0 = (i0 + i4) * (1 << kConstBits), t1 = (i0 - i4) * (1 << kConstBits);
  const int64_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  int64_t a0 = i7, a1 = i5, a2 = i3, a3 = i1;
  z1 = a0 + a3;
  int64_t z2 = a1 + a2, z3 = a0 + a2, z4 = a1 + a3;
  const int64_t z5 = (z3 + z4) * kF1175;
  a0 *= kF0298; a1 *= kF2053; a2 *= kF3072; a3 *= kF1501;
  z1 *= -kF0899; z2 *= -kF2562; z3 *= -kF1961; z4 *= -kF0390;
  z3 += z5; z4 += z5;
  a0 += z1 + z3; a1 += z2 + z4; a2 += z2 + z3; a3 += z1 + z4;
  o[0] = t10 + a3; o[7] = t10 - a3; o[1] = t11 + a2; o[6] = t11 - a2;
  o[2] = t12 + a1; o[5] = t12 - a1; o[3] = t13 + a0; o[4] = t13 - a0;
}

// one block: coefficients (natural order) x qt -> 8 x 8 samples at out (row stride `stride`)
MFR_HD void idct_block(const int16_t* in, const int32_t* qt, uint8_t* out, int stride) {
  int32_t ws[64];
  for (int c = 0; c < 8; ++c) {     // pass 1: columns; all-zero AC gives dc << PASS1_BITS, which the full pass equals
    int32_t q[8];
    int64_t o[8];
    for (int r = 0; r < 8; ++r) q[r] = static_cast<int32_t>(in[r * 8 + c]) * qt[r * 8 + c];
    idct_1d(q[0], q[1], q[2], q[3], q[4], q[5], q[6], q[7], o);
    for (int r = 0; r < 8; ++r) ws[r * 8 + c] = static_cast<int32_t>(descale(o[r], kConstBits - kPass1Bits));
  }
  for (int r = 0; r < 8; ++r) {     // pass 2: rows (libjpeg's zero-row shortcut is the same arithmetic)
    const int32_t* w = ws + r * 8;
    int64_t o[8];
    idct_1d(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7], o);
    for (int x = 0; x < 8; ++x) out[r * stride + x] = idct_limit(descale(o[x], kConstBits + kPass1Bits + 3));
  }
}

// ------------------------------------------------------------------------------------------ upsample, colour, orientation
// source pixel (x, y) of output pixel (ox, oy) under Exif orientation o (cv2's ExifTransform: flips / transposes)
MFR_HD void orient_src(int o, int w, int h, int ox, int oy, int& x, int& y) {
  switch (o) {
    case 2: x = w - 1 - ox; y = oy; break;               // mirror horizontal
    case 3: x = w - 1 - ox; y = h - 1 - oy; break;       // rotate 180
    case 4: x = ox; y = h - 1 - oy; break;               // mirror vertical
    case 5: x = oy; y = ox; break;                       // transpose
    case 6: x = oy; y = h - 1 - ox; break;               // rotate 90 clockwise
    case 7: x = w - 1 - oy; y = h - 1 - ox; break;       // transverse
    case 8: x = w - 1 - oy; y = ox; break;               // rotate 90 counter-clockwise
    default: x = ox; y = oy; break;
  }
}

// Chroma sample of component c at full-resolution pixel (x, y): libjpeg's fancy upsampling. h2v1: (3 s[j] + s[j -+ 1]
// + 1 / 2) >> 2 for the left / right output of s[j]; h2v2: column sums 3 s[i][j] + s[i -+ 1][j] (context rows replicate
// the first / last row), then (3 cs[j] + cs[j -+ 1] + 8 / 7) >> 4. Neighbours past the first / last column replicate it,
// which is what libjpeg's edge cases compute. A plane of at most 2 samples per row is replicated instead (libjpeg-turbo
// selects fancy upsampling only for downsampled_width > 2).
MFR_HD int chroma(const Desc& d, const uint8_t* planes, int c, int x, int y) {
  const Comp& cp = d.comp[c];
  const uint8_t* p = planes + cp.plane;
  const int stride = cp.bw * 8;
  if (d.hmax == 1) return p[y * stride + x];            // 4:4:4
  if (cp.dw <= 2) return p[(y / d.vmax) * stride + (x >> 1)];
  const int j = x >> 1, right = x & 1;
  const int jn = right ? (j + 1 < cp.dw ? j + 1 : cp.dw - 1) : (j > 0 ? j - 1 : 0);
  if (d.vmax == 1) {                                     // h2v1
    const uint8_t* row = p + y * stride;
    return (3 * row[j] + row[jn] + (right ? 2 : 1)) >> 2;
  }
  const int i = y >> 1;                                  // h2v2
  const int in = (y & 1) ? (i + 1 < cp.dh ? i + 1 : cp.dh - 1) : (i > 0 ? i - 1 : 0);
  const uint8_t* r0 = p + i * stride;
  const uint8_t* r1 = p + in * stride;
  const int cs = 3 * r0[j] + r1[j], csn = 3 * r0[jn] + r1[jn];
  return (3 * cs + csn + (right ? 7 : 8)) >> 4;
}

MFR_HD uint8_t clamp255(int v) { return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// output pixel (ox, oy): gray = the Y plane as coded; RGB = jdcolor's ycc_rgb_convert (SCALEBITS 16, ONE_HALF rounding)
// of the upsampled planes, or Y replicated for a one-component file
MFR_HD void pixel(const Desc& d, const uint8_t* planes, int ox, int oy, uint8_t* out) {
  int x, y;
  orient_src(d.orient, d.width, d.height, ox, oy, x, y);
  const int Y = planes[d.comp[0].plane + static_cast<long long>(y) * d.comp[0].bw * 8 + x];
  if (!d.rgb) { out[0] = static_cast<uint8_t>(Y); return; }
  if (d.ncomp == 1) { out[0] = out[1] = out[2] = static_cast<uint8_t>(Y); return; }
  const int cb = chroma(d, planes, 1, x, y) - 128, cr = chroma(d, planes, 2, x, y) - 128;
  constexpr int32_t kHalf = 1 << 15;
  constexpr int32_t kCrR = 91881, kCbB = 116130, kCrG = 46802, kCbG = 22554;   // FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414)
  out[0] = clamp255(Y + ((kCrR * cr + kHalf) >> 16));
  out[1] = clamp255(Y + ((-kCbG * cb + kHalf - kCrG * cr) >> 16));
  out[2] = clamp255(Y + ((kCbB * cb + kHalf) >> 16));
}

}  // namespace jpeg
}  // namespace mfr
