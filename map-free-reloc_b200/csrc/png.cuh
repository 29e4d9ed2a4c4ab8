// Gray PNG decode (colour type 0, 8- or 16-bit, non-interlaced): the arithmetic of cv2.imread(IMREAD_UNCHANGED) on
// the depth maps the reference reads (lib/datasets/utils.py:77-81). RFC 1950 (zlib) + RFC 1951 (deflate) + the PNG
// row filters, CRC-32 and Adler-32 as MFR_HD functions, so that the kernels of image_io.cu and the serial CPU hook
// mfr_host_png_decode run one copy of them. The host parser (image_io.cu) has validated the chunk structure and the
// zlib header; everything below bound-checks the compressed data, which it treats as untrusted.
#pragma once

#include <stdint.h>

#ifndef MFR_HD
#ifdef __CUDACC__
#define MFR_HD __host__ __device__ __forceinline__
#else
#define MFR_HD inline
#endif
#endif
#ifdef __CUDACC__
#define MFR_HDC __host__ __device__ constexpr
#else
#define MFR_HDC constexpr
#endif

namespace mfr {
namespace png {

// ------------------------------------------------------------------------------------------ CRC-32 (ISO 3309, reflected)
constexpr uint32_t kCrcPoly = 0xEDB88320u;

struct CrcTables {
  uint32_t byte[256];   // register update of one byte
  uint32_t x2n[32];     // x^(2^k) mod P, for shifting a register over n zero bytes
};

// a * b mod P in the reflected representation (bit 31 = x^0)
MFR_HDC uint32_t multmodp(uint32_t a, uint32_t b) {
  uint32_t m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = (b & 1) ? (b >> 1) ^ kCrcPoly : b >> 1;
  }
  return p;
}

constexpr CrcTables make_crc_tables() {
  CrcTables t{};
  for (uint32_t i = 0; i < 256; ++i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ kCrcPoly : c >> 1;
    t.byte[i] = c;
  }
  uint32_t p = 1u << 30;   // x^1
  for (int k = 0; k < 32; ++k) {
    t.x2n[k] = p;
    p = multmodp(p, p);
  }
  return t;
}

// register after `n` more bytes (no pre / post inversion: crc32(d) = ~crc_update(0xFFFFFFFF, d))
MFR_HD uint32_t crc_update(const uint32_t* table, uint32_t reg, const uint8_t* p, uint32_t n) {
  for (uint32_t i = 0; i < n; ++i) reg = (reg >> 8) ^ table[(reg ^ p[i]) & 0xFF];
  return reg;
}

// register shifted over n zero bytes: reg * x^(8n) mod P. crc_update(r, A || B) = crc_shift(crc_update(r, A), |B|) ^
// crc_update(0, B), which is how the CRC kernel joins the pieces of a long chunk.
MFR_HD uint32_t crc_shift(const uint32_t* x2n, uint32_t reg, uint32_t n) {
  uint32_t p = 1u << 31;   // x^0
  for (int k = 3; n; n >>= 1, ++k)
    if (n & 1) p = multmodp(x2n[k & 31], p);
  return multmodp(p, reg);
}

// ------------------------------------------------------------------------------------------ Adler-32
constexpr uint32_t kAdlerMod = 65521;

// Adler-32 of n bytes from S1 = sum of the bytes and S2 = sum of position * byte (positions from 0, any order of
// accumulation): a = 1 + S1, b = n + n S1 - S2 (mod 65521)
MFR_HD uint32_t adler_from_sums(uint64_t n, uint64_t s1, uint64_t s2) {
  const uint64_t M = kAdlerMod, nm = n % M, s1m = s1 % M, s2m = s2 % M;
  const uint64_t a = (1 + s1m) % M;
  const uint64_t b = (nm + nm * s1m % M + M - s2m) % M;
  return static_cast<uint32_t>((b << 16) | a);
}

// ------------------------------------------------------------------------------------------ inflate (RFC 1951)
// Decode-table entry (uint32): value [0,16) | code length [16,20) | extra bits [20,24) | kind [24,27).
// Codes of up to kRootBits bits resolve in the root table. The canonical codes longer than kRootBits take the top of
// the code space: their kRootBits-bit prefixes ("regions") are the consecutive values first_long .. 2^kRootBits - 1.
// The root entry of a region links to its subtable of 2^(L - kRootBits) entries, L the longest code in the region.
constexpr int kRootBits = 10;
// Root + subtables always fit: a region with a 2^k-entry subtable holds at least k + 1 codes (a complete code fills
// it), so the subtables of <= 286 codes take at most 286 * max_k 2^k / (k + 1) = 286 * 32 / 6 < 1526 entries.
constexpr int kTableCap = (1 << kRootBits) + 1536;
constexpr int kMaxRegions = 288;  // at most one region per long code
enum : uint32_t { kLit = 0, kLen = 1, kEnd = 2, kBad = 3, kLink = 4, kDist = 5 };

MFR_HD uint32_t entry(uint32_t kind, uint32_t value, uint32_t nbits, uint32_t extra) {
  return value | (nbits << 16) | (extra << 20) | (kind << 24);
}
MFR_HD uint32_t e_kind(uint32_t e) { return e >> 24; }
MFR_HD uint32_t e_bits(uint32_t e) { return (e >> 16) & 15; }
MFR_HD uint32_t e_extra(uint32_t e) { return (e >> 20) & 15; }
MFR_HD uint32_t e_value(uint32_t e) { return e & 0xFFFF; }

// RFC 1951 3.2.5's base / extra-bit tables in closed form: length symbol 257 + s, distance symbol s
MFR_HD uint32_t len_extra(int s) { return s < 8 || s == 28 ? 0 : (s - 4) >> 2; }
MFR_HD uint32_t len_base(int s) { return s < 8 ? 3 + s : (s == 28 ? 258 : ((4u + (s & 3)) << len_extra(s)) + 3); }
MFR_HD uint32_t dist_extra(int s) { return s < 4 ? 0 : (s - 2) >> 1; }
MFR_HD uint32_t dist_base(int s) { return s < 4 ? 1 + s : ((2u + (s & 1)) << dist_extra(s)) + 1; }

MFR_HD uint32_t rev_bits(uint32_t c, int n) {
  uint32_t r = 0;
  for (int i = 0; i < n; ++i, c >>= 1) r = (r << 1) | (c & 1);
  return r;
}

// Table layout of one code from its code lengths: per symbol its bit-reversed canonical code (codes[]), and per region
// its subtable (region[i] = offset | bits << 16 for region first_long + i). Returns 0, or 1 for an over-subscribed code
// or an incomplete one (allowed, as zlib allows it, only for a single code of length 1, or for no codes at all).
struct Layout {
  uint32_t first_long;
  uint32_t* region;   // kMaxRegions entries
};
MFR_HD int huff_layout(const uint8_t* lens, int n, uint16_t* codes, Layout& lay) {
  const int R = kRootBits;
  int count[16] = {0};
  for (int s = 0; s < n; ++s) count[lens[s]]++;
  count[0] = 0;
  int max = 0, left = 1;
  for (int l = 1; l <= 15; ++l) {
    if (count[l]) max = l;
    left = (left << 1) - count[l];
    if (left < 0) return 1;                              // over-subscribed
  }
  if (left > 0 && max != 1 && max != 0) return 1;       // incomplete
  int next[16];
  next[1] = 0;
  for (int l = 1; l < 15; ++l) next[l + 1] = (next[l] + count[l]) << 1;
  lay.first_long = static_cast<uint32_t>(next[R] + count[R]);
  if (max > R) {
    const uint32_t nreg = (1u << R) - lay.first_long;    // complete code: every region holds a long code
    if (nreg > kMaxRegions) return 1;
    for (int l = R + 1; l <= max; ++l)                   // ascending lengths: the last write is the region's longest
      if (count[l]) {
        const uint32_t r0 = static_cast<uint32_t>(next[l]) >> (l - R), r1 = static_cast<uint32_t>(next[l] + count[l] - 1) >> (l - R);
        for (uint32_t r = r0; r <= r1; ++r) lay.region[r - lay.first_long] = static_cast<uint32_t>(l - R);
      }
    uint32_t off = 1u << R;
    for (uint32_t i = 0; i < nreg; ++i) {
      const uint32_t bits = lay.region[i];
      lay.region[i] = off | (bits << 16);
      off += 1u << bits;
    }
    if (off > static_cast<uint32_t>(kTableCap)) return 1;   // cannot happen for a complete code (see kTableCap)
  }
  for (int s = 0; s < n; ++s)
    codes[s] = lens[s] ? static_cast<uint16_t>(rev_bits(static_cast<uint32_t>(next[lens[s]]++), lens[s])) : 0;
  return 0;
}

// Entry of symbol s of a literal / length table (dist = 0) or a distance table (dist = 1)
MFR_HD uint32_t sym_entry(int s, int len, int dist) {
  if (dist) return s < 30 ? entry(kDist, dist_base(s), len, dist_extra(s)) : entry(kBad, 0, len, 0);
  if (s < 256) return entry(kLit, s, len, 0);
  if (s == 256) return entry(kEnd, 0, len, 0);
  if (s < 286) return entry(kLen, len_base(s - 257), len, len_extra(s - 257));
  return entry(kBad, 0, len, 0);
}

// Fills the table from huff_layout's codes: lane `lane` of `nlanes` writes its share (a warp, or 1 lane on the host).
// Step 1 marks every entry invalid; the caller orders step 1 before step 2 (__syncwarp) when nlanes > 1.
MFR_HD void huff_fill_invalid(uint32_t* t, int lane, int nlanes) {
  for (int i = lane; i < kTableCap; i += nlanes) t[i] = entry(kBad, 0, 1, 0);
}
// Step 2: each lane's symbols, and for a long code the link of its region (the same entry from every code in it).
MFR_HD void huff_fill(const uint8_t* lens, const uint16_t* codes, int n, int dist, const Layout& lay, uint32_t* t,
                      int lane, int nlanes) {
  const int R = kRootBits;
  for (int s = lane; s < n; s += nlanes) {
    const int l = lens[s];
    if (!l) continue;
    const uint32_t e = sym_entry(s, l, dist);
    if (l <= R) {
      for (uint32_t i = codes[s]; i < (1u << R); i += 1u << l) t[i] = e;
    } else {
      const uint32_t pre = codes[s] & ((1u << R) - 1);
      const uint32_t sub = lay.region[rev_bits(pre, R) - lay.first_long], off = sub & 0xFFFF, sb = sub >> 16;
      t[pre] = entry(kLink, off, sb, 0);
      for (uint32_t i = codes[s] >> R; i < (1u << sb); i += 1u << (l - R)) t[off + i] = e;
    }
  }
}

// Step 3 (after step 2, ordered by the caller as step 1 before 2): pair[i] for root index i = two literals whose codes
// both lie within the index's kRootBits bits, as lit0 | lit1 << 8 | total bits << 16, else 0. One lookup then emits
// two literals, which halves the serial lookup chain on literal-heavy data.
MFR_HD void huff_fill_pairs(const uint32_t* lit, uint32_t* pair, int lane, int nlanes) {
  const int R = kRootBits;
  for (int i = lane; i < (1 << R); i += nlanes) {
    const uint32_t e1 = lit[i];
    uint32_t v = 0;
    if (e_kind(e1) == kLit) {
      const uint32_t l1 = e_bits(e1);
      const uint32_t e2 = lit[static_cast<uint32_t>(i) >> l1];   // the unknown high bits are zero: valid when l2 <= R - l1
      if (e_kind(e2) == kLit && e_bits(e2) <= R - l1) v = e_value(e1) | (e_value(e2) << 8) | ((l1 + e_bits(e2)) << 16);
    }
    pair[i] = v;
  }
}

// Bit reader (LSB first) over a stream of `len` bytes held in 4-byte aligned words. The next word is loaded one refill
// ahead, so that its load overlaps the symbols decoded from the current one. Words past the stream read as zero; the
// end check compares the bits consumed with the stream.
MFR_HD uint32_t load_word(const uint32_t* w, uint32_t i, uint32_t nw) {
#ifdef __CUDA_ARCH__
  return i < nw ? __ldg(w + i) : 0u;
#else
  return i < nw ? w[i] : 0u;
#endif
}
struct Bits {
  const uint32_t* w;
  uint32_t len, nw;    // stream bytes, words holding them
  uint32_t wi, pre;    // pre = word wi, the next one to enter acc
  uint64_t acc;
  int n;
  MFR_HD void seek(uint32_t byte) {
    wi = byte >> 2;
    const int sh = static_cast<int>(byte & 3) * 8;
    acc = load_word(w, wi, nw) >> sh;
    n = 32 - sh;
    pre = load_word(w, ++wi, nw);
  }
  MFR_HD void refill() {
    if (n >= 32) return;
    acc |= static_cast<uint64_t>(pre) << n;
    n += 32;
    pre = load_word(w, ++wi, nw);
  }
  MFR_HD uint32_t peek(int k) const { return static_cast<uint32_t>(acc) & ((1u << k) - 1u); }
  MFR_HD void drop(int k) { acc >>= k; n -= k; }
  MFR_HD uint64_t consumed() const { return static_cast<uint64_t>(wi) * 32 - n; }
  MFR_HD bool overrun() const { return consumed() > static_cast<uint64_t>(len) * 8; }
};

MFR_HD uint32_t lookup(const uint32_t* t, uint32_t bits) {
  uint32_t e = t[bits & ((1u << kRootBits) - 1)];
  if (e_kind(e) == kLink) e = t[e_value(e) + ((bits >> kRootBits) & ((1u << e_bits(e)) - 1))];
  return e;
}

enum Cmd : int { kCmdMatch = 1, kCmdStored, kCmdBuild, kCmdFlush, kCmdDone, kCmdError };

// The decoder state. Output goes to a window win[pos & wmask]: on the device a shared-memory ring that the warp
// flushes to the output (kCmdFlush once flush_at bytes are pending), on the host the whole output buffer.
struct Inflate {
  Bits br;
  uint8_t* win;
  uint32_t wmask, out, flushed, flush_at, total, window;   // window: 1 << wbits of the zlib header
  int mode;                                                // 0: block header, 1: Huffman codes, 2: stored bytes
  int last, fixed;                                         // fixed: the tables hold the fixed code
  uint32_t stored_left, stored_pos;                        // stored block: bytes left, their stream offset
  uint32_t cmd_len, cmd_dist, cmd_out;                     // match / stored copy handed to the caller
  int nlen, ndist;                                         // kCmdBuild: lens[0, nlen) litlen, lens[nlen, nlen + ndist) dist
};

MFR_HD void inflate_init(Inflate& s, const uint32_t* deflate, uint32_t len, uint8_t* win, uint32_t wmask, uint32_t flush_at,
                         uint32_t total, int wbits) {
  s.br.w = deflate; s.br.len = len; s.br.nw = (len + 3) / 4;
  s.br.seek(0);
  s.win = win; s.wmask = wmask; s.out = 0; s.flushed = 0; s.flush_at = flush_at; s.total = total;
  s.window = 1u << wbits;
  s.mode = 0; s.last = 0; s.fixed = 0; s.stored_left = 0; s.stored_pos = 0;
  s.cmd_len = s.cmd_dist = s.cmd_out = 0; s.nlen = s.ndist = 0;
}

// Copies a match of `len` bytes from `dist` back within the window (serial; the warp kernel copies long ones itself).
MFR_HD void copy_match(uint8_t* win, uint32_t wmask, uint32_t out, uint32_t len, uint32_t dist) {
  if (dist == 1) {
    const uint8_t b = win[(out - 1) & wmask];
    for (uint32_t i = 0; i < len; ++i) win[(out + i) & wmask] = b;
  } else {
    for (uint32_t i = 0; i < len; ++i) win[(out + i) & wmask] = win[(out + i - dist) & wmask];
  }
}

// Reads a dynamic block's code lengths into lens (19-symbol code-length code through a small table); 0 or 1 on error.
MFR_HD int read_dynamic(Inflate& s, uint8_t* lens) {
  Bits& b = s.br;
  b.refill();
  const int nlen = static_cast<int>(b.peek(5)) + 257, ndist = static_cast<int>((b.acc >> 5) & 31) + 1,
            ncode = static_cast<int>((b.acc >> 10) & 15) + 4;
  b.drop(14);
  if (nlen > 286 || ndist > 30) return 1;
  const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
  uint8_t cl[19] = {0};
  for (int i = 0; i < ncode; ++i) {
    b.refill();
    cl[order[i]] = static_cast<uint8_t>(b.peek(3));
    b.drop(3);
  }
  // code-length code: 7-bit direct table, (len << 5) | symbol, 0 = no code
  int count[8] = {0};
  for (int i = 0; i < 19; ++i) count[cl[i]]++;
  count[0] = 0;
  int left = 1, max = 0;
  for (int l = 1; l <= 7; ++l) {
    if (count[l]) max = l;
    left = (left << 1) - count[l];
    if (left < 0) return 1;
  }
  if (left > 0 && max != 1) return 1;                    // incomplete code-length codes are invalid (zlib: CODES)
  uint8_t tbl[128] = {0};
  int next[8];
  next[1] = 0;
  for (int l = 1; l < 7; ++l) next[l + 1] = (next[l] + count[l]) << 1;
  for (int sym = 0; sym < 19; ++sym) {
    const int l = cl[sym];
    if (!l) continue;
    const uint32_t c = rev_bits(static_cast<uint32_t>(next[l]++), l);
    for (uint32_t i = c; i < 128; i += 1u << l) tbl[i] = static_cast<uint8_t>((l << 5) | sym);
  }
  int i = 0;
  while (i < nlen + ndist) {
    b.refill();
    const uint8_t e = tbl[b.peek(7)];
    if (!e) return 1;
    b.drop(e >> 5);
    const int sym = e & 31;
    if (sym < 16) { lens[i++] = static_cast<uint8_t>(sym); continue; }
    int rep, val = 0;
    if (sym == 16) {
      if (i == 0) return 1;
      val = lens[i - 1];
      rep = 3 + static_cast<int>(b.peek(2)); b.drop(2);
    } else if (sym == 17) {
      rep = 3 + static_cast<int>(b.peek(3)); b.drop(3);
    } else {
      rep = 11 + static_cast<int>(b.peek(7)); b.drop(7);
    }
    if (i + rep > nlen + ndist) return 1;
    while (rep--) lens[i++] = static_cast<uint8_t>(val);
  }
  if (lens[256] == 0) return 1;                          // no end-of-block code
  if (b.overrun()) return 1;
  s.nlen = nlen;
  s.ndist = ndist;
  return 0;
}

// Runs the decoder until it needs its caller: a table build (lens / codes / layouts filled), a long match or a stored
// run to copy (cmd_out, cmd_len, cmd_dist; s.out already advanced past it), a flush, the end, or an error. Matches
// shorter than `warp_len` and literals are written here.
MFR_HD int inflate_run(Inflate& s, const uint32_t* lit, const uint32_t* pair, const uint32_t* dst, uint8_t* lens, uint16_t* codes,
                       Layout* lay, uint32_t warp_len) {
  Bits& b = s.br;
  for (;;) {
    if (s.out - s.flushed >= s.flush_at) return kCmdFlush;
    if (s.mode == 1) {
      b.refill();
      const uint32_t pe = pair[b.peek(kRootBits)];
      if (pe) {
        if (s.total - s.out < 2) return kCmdError;       // more data than the image holds
        s.win[s.out & s.wmask] = static_cast<uint8_t>(pe);
        s.win[(s.out + 1) & s.wmask] = static_cast<uint8_t>(pe >> 8);
        s.out += 2;
        b.drop(static_cast<int>(pe >> 16));
        continue;
      }
      uint32_t e = lookup(lit, b.peek(15));
      uint32_t k = e_kind(e);
      b.drop(static_cast<int>(e_bits(e)));
      if (k == kLit) {
        if (s.out >= s.total) return kCmdError;          // more data than the image holds
        s.win[s.out & s.wmask] = static_cast<uint8_t>(e_value(e));
        ++s.out;
        continue;
      }
      if (k == kLen) {
        const int xb = static_cast<int>(e_extra(e));
        const uint32_t len = e_value(e) + b.peek(xb);
        b.drop(xb);
        b.refill();
        e = lookup(dst, b.peek(15));
        if (e_kind(e) != kDist) return kCmdError;
        b.drop(static_cast<int>(e_bits(e)));
        const int xd = static_cast<int>(e_extra(e));
        const uint32_t dist = e_value(e) + b.peek(xd);
        b.drop(xd);
        if (dist > s.out || dist > s.window || len > s.total - s.out) return kCmdError;
        if (b.overrun()) return kCmdError;
        if (len >= warp_len) {
          s.cmd_out = s.out; s.cmd_len = len; s.cmd_dist = dist;
          s.out += len;
          return kCmdMatch;
        }
        copy_match(s.win, s.wmask, s.out, len, dist);
        s.out += len;
        continue;
      }
      if (k == kEnd) {
        if (b.overrun()) return kCmdError;
        s.mode = 0;
        if (s.last) {
          const uint64_t bytes = (b.consumed() + 7) / 8;   // the Adler-32 trailer follows at the next byte
          return bytes == b.len && s.out == s.total ? kCmdDone : kCmdError;
        }
        continue;
      }
      return kCmdError;                                  // invalid code
    }
    if (s.mode == 2) {
      if (s.stored_left == 0) {
        b.seek(s.stored_pos);
        s.mode = 0;
        if (s.last) return s.stored_pos == b.len && s.out == s.total ? kCmdDone : kCmdError;
        continue;
      }
      const uint32_t n = s.stored_left < 4096u ? s.stored_left : 4096u;
      if (n > b.len - s.stored_pos || n > s.total - s.out) return kCmdError;
      s.cmd_out = s.out; s.cmd_len = n; s.cmd_dist = s.stored_pos;
      s.stored_pos += n; s.out += n; s.stored_left -= n;
      return kCmdStored;
    }
    // block header
    b.refill();
    s.last = static_cast<int>(b.peek(1));
    const uint32_t type = (static_cast<uint32_t>(b.acc) >> 1) & 3;
    b.drop(3);
    if (type == 0) {
      b.drop(b.n & 7);                                   // to the byte boundary
      b.refill();
      const uint32_t len = b.peek(16), nlen = static_cast<uint32_t>(b.acc >> 16) & 0xFFFF;
      b.drop(32);
      if (len != (~nlen & 0xFFFF) || b.overrun()) return kCmdError;
      s.stored_left = len;
      s.stored_pos = static_cast<uint32_t>(b.consumed() / 8);
      s.mode = 2;
      continue;
    }
    if (type == 1) {
      s.mode = 1;
      if (s.fixed) continue;
      for (int i = 0; i < 144; ++i) lens[i] = 8;
      for (int i = 144; i < 256; ++i) lens[i] = 9;
      for (int i = 256; i < 280; ++i) lens[i] = 7;
      for (int i = 280; i < 288; ++i) lens[i] = 8;
      for (int i = 0; i < 32; ++i) lens[288 + i] = 5;
      s.nlen = 288; s.ndist = 32;
    } else if (type == 2) {
      if (read_dynamic(s, lens)) return kCmdError;
      s.mode = 1;
    } else {
      return kCmdError;                                  // block type 3
    }
    if (huff_layout(lens, s.nlen, codes, lay[0]) || huff_layout(lens + s.nlen, s.ndist, codes + s.nlen, lay[1]))
      return kCmdError;
    s.fixed = type == 1;
    return kCmdBuild;
  }
}

// ------------------------------------------------------------------------------------------ row filters, output
MFR_HD uint8_t paeth(int a, int b, int c) {
  const int p = a + b - c;
  const int pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
  return static_cast<uint8_t>(pa <= pb && pa <= pc ? a : (pb <= pc ? b : c));
}

// Unfilters one row in place: cur = the row's bytes after its filter byte, prev = the previous row unfiltered
// (nullptr for the first row). Returns 1 for a filter type > 4.
MFR_HD int unfilter_row(int f, uint8_t* cur, const uint8_t* prev, uint32_t rb, int bpp) {
  switch (f) {
    case 0: return 0;
    case 1:
      for (uint32_t i = bpp; i < rb; ++i) cur[i] = static_cast<uint8_t>(cur[i] + cur[i - bpp]);
      return 0;
    case 2:
      if (prev) for (uint32_t i = 0; i < rb; ++i) cur[i] = static_cast<uint8_t>(cur[i] + prev[i]);
      return 0;
    case 3:
      for (uint32_t i = 0; i < rb; ++i) {
        const int a = i >= static_cast<uint32_t>(bpp) ? cur[i - bpp] : 0, up = prev ? prev[i] : 0;
        cur[i] = static_cast<uint8_t>(cur[i] + ((a + up) >> 1));
      }
      return 0;
    case 4:
      for (uint32_t i = 0; i < rb; ++i) {
        const bool l = i >= static_cast<uint32_t>(bpp);
        const int a = l ? cur[i - bpp] : 0, up = prev ? prev[i] : 0, c = (l && prev) ? prev[i - bpp] : 0;
        cur[i] = static_cast<uint8_t>(cur[i] + paeth(a, up, c));
      }
      return 0;
    default: return 1;
  }
}

// Output kind 0: the samples as stored (16-bit big-endian -> native, as libpng with png_set_swap); kind 1: float32
// v / 1000 rounded from double (read_depth_image: NumPy's float64 division, then .float()).
MFR_HD void store_sample(const uint8_t* row, int x, int depth, int kind, void* dst, uint64_t idx) {
  const uint32_t v = depth == 16 ? (static_cast<uint32_t>(row[2 * x]) << 8) | row[2 * x + 1] : row[x];
  if (kind == 1) static_cast<float*>(dst)[idx] = static_cast<float>(static_cast<double>(v) / 1000.0);
  else if (depth == 16) static_cast<uint16_t*>(dst)[idx] = static_cast<uint16_t>(v);
  else static_cast<uint8_t*>(dst)[idx] = static_cast<uint8_t>(v);
}

}  // namespace png
}  // namespace mfr
