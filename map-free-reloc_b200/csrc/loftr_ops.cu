// SIMT kernels of the LoFTR matcher (everything that is not a GEMM). See loftr_ops.cuh.
#include "loftr_ops.cuh"

#include <algorithm>
#include <cstring>

namespace mfr {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------ stem
constexpr int kStemPx = 32;
__device__ __forceinline__ unsigned short f2bf(float f) {
  unsigned short r;
  asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(f));
  return r;
}
__device__ __forceinline__ float bf2f(unsigned short b) { return __uint_as_float(static_cast<unsigned>(b) << 16); }

template <bool OBF>
__global__ void __launch_bounds__(128) stem_kernel(const float* __restrict__ img,
                                                   const float* __restrict__ w,
                                                   const float* __restrict__ bias,
                                                   float* __restrict__ out, int H, int W, int Ho,
                                                   int Wo) {
  __shared__ float patch[7][2 * kStemPx + 8];
  const int n = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * kStemPx;
  const int c = threadIdx.x;
  constexpr int PW = 2 * kStemPx + 5;
  for (int idx = threadIdx.x; idx < 7 * PW; idx += 128) {
    const int ky = idx / PW, kx = idx - ky * PW;
    const int iy = 2 * y - 3 + ky, ix = 2 * x0 - 3 + kx;
    float v = 0.f;
    if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = img[(static_cast<size_t>(n) * H + iy) * W + ix];
    patch[ky][kx] = v;
  }
  float wr[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) wr[k] = w[c * 49 + k];
  const float b = bias[c];
  __syncthreads();
  for (int px0 = 0; px0 < kStemPx; px0 += 8) {
    float acc[8];
#pragma unroll
    for (int p = 0; p < 8; ++p) acc[p] = 0.f;
#pragma unroll
    for (int ky = 0; ky < 7; ++ky) {
      float row[21];
#pragma unroll
      for (int j = 0; j < 21; ++j) row[j] = patch[ky][2 * px0 + j];
#pragma unroll
      for (int kx = 0; kx < 7; ++kx)
#pragma unroll
        for (int p = 0; p < 8; ++p) acc[p] = fmaf(wr[ky * 7 + kx], row[2 * p + kx], acc[p]);
    }
#pragma unroll
    for (int p = 0; p < 8; ++p) {
      const int x = x0 + px0 + p;
      if (x < Wo) {
        const size_t o = ((static_cast<size_t>(n) * Ho + y) * Wo + x) * 128 + c;
        if constexpr (OBF) reinterpret_cast<unsigned short*>(out)[o] = f2bf(fmaxf(acc[p] + b, 0.f));
        else out[o] = fmaxf(acc[p] + b, 0.f);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ upsample
template <bool SBF>
__device__ __forceinline__ float4 ld4(const void* base, size_t elem) {
  if constexpr (SBF) {
    const uint2 u = *reinterpret_cast<const uint2*>(reinterpret_cast<const unsigned short*>(base) + elem);
    return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                       __uint_as_float(u.y & 0xffff0000u));
  } else {
    return *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(base) + elem);
  }
}
// dst[n,y,x,c] += bilinear(src)[n,y,x,c]; pixel strides lds / ldd (elements), C4 = C / 4
template <bool SBF, bool DBF>
__global__ void upsample2x_add_kernel(const void* __restrict__ src, void* __restrict__ dst, int N, int Hs, int Ws,
                                      int C4, int lds, int ldd, float ry, float rx) {
  const int Hd = 2 * Hs, Wd = 2 * Ws;
  const size_t total = static_cast<size_t>(N) * Hd * Wd * C4;
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c4 = static_cast<int>(idx % C4);
  size_t pix = idx / C4;
  const size_t dpix = pix;
  const int x = static_cast<int>(pix % Wd);
  pix /= Wd;
  const int y = static_cast<int>(pix % Hd);
  const int n = static_cast<int>(pix / Hd);
  const float sy = ry * y, sx = rx * x;
  const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
  const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const size_t sb = static_cast<size_t>(n) * Hs * Ws;
  const float4 a = ld4<SBF>(src, (sb + static_cast<size_t>(y0) * Ws + x0) * lds + c4 * 4);
  const float4 b = ld4<SBF>(src, (sb + static_cast<size_t>(y0) * Ws + x1) * lds + c4 * 4);
  const float4 c = ld4<SBF>(src, (sb + static_cast<size_t>(y1) * Ws + x0) * lds + c4 * 4);
  const float4 d = ld4<SBF>(src, (sb + static_cast<size_t>(y1) * Ws + x1) * lds + c4 * 4);
  const size_t de = dpix * ldd + c4 * 4;
  float4 v = ld4<DBF>(dst, de);
  v.x += hy * (hx * a.x + lx * b.x) + ly * (hx * c.x + lx * d.x);
  v.y += hy * (hx * a.y + lx * b.y) + ly * (hx * c.y + lx * d.y);
  v.z += hy * (hx * a.z + lx * b.z) + ly * (hx * c.z + lx * d.z);
  v.w += hy * (hx * a.w + lx * b.w) + ly * (hx * c.w + lx * d.w);
  if constexpr (DBF) {
    uint2 o;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.x) : "f"(v.y), "f"(v.x));
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(o.y) : "f"(v.w), "f"(v.z));
    *reinterpret_cast<uint2*>(reinterpret_cast<unsigned short*>(dst) + de) = o;
  } else {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(dst) + de) = v;
  }
}

// Same op for a bf16 destination, 8 channels (16 bytes of dst) per thread; grid (ceil(Wd*C8/256), Hd, N), no 64-bit
// divisions. C8 = ceil(C / 8): the pad channels of a 200-stride 196-channel map are read and written as zeros.
__device__ __forceinline__ void ld8(const void* p, size_t e, bool bf, float (&o)[8]) {
  if (bf) {
    const uint4 u = *reinterpret_cast<const uint4*>(static_cast<const unsigned short*>(p) + e);
    const unsigned w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) { o[2 * k] = __uint_as_float(w[k] << 16); o[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u); }
  } else {
    const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + e);
    const float4 b = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + e + 4);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
  }
}
template <bool SBF>
__global__ void __launch_bounds__(256) upsample2x_add8_kernel(const void* __restrict__ src, void* __restrict__ dst, int Hs,
                                                              int Ws, int C8, int lds, int ldd, float ry, float rx) {
  const int Hd = 2 * Hs, Wd = 2 * Ws;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= Wd * C8) return;
  const int x = idx / C8, c8 = idx - x * C8;
  const int y = blockIdx.y, n = blockIdx.z;
  const float sy = ry * y, sx = rx * x;
  const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
  const int y1 = y0 + (y0 < Hs - 1 ? 1 : 0), x1 = x0 + (x0 < Ws - 1 ? 1 : 0);
  const float ly = sy - y0, lx = sx - x0;
  const float hy = 1.f - ly, hx = 1.f - lx;
  const size_t sb = static_cast<size_t>(n) * Hs * Ws;
  float a[8], b[8], c[8], d[8], v[8];
  ld8(src, (sb + static_cast<size_t>(y0) * Ws + x0) * lds + c8 * 8, SBF, a);
  ld8(src, (sb + static_cast<size_t>(y0) * Ws + x1) * lds + c8 * 8, SBF, b);
  ld8(src, (sb + static_cast<size_t>(y1) * Ws + x0) * lds + c8 * 8, SBF, c);
  ld8(src, (sb + static_cast<size_t>(y1) * Ws + x1) * lds + c8 * 8, SBF, d);
  const size_t de = ((static_cast<size_t>(n) * Hd + y) * Wd + x) * ldd + c8 * 8;
  ld8(dst, de, true, v);
  uint4 o;
  unsigned* ow = reinterpret_cast<unsigned*>(&o);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float r0 = v[2 * k] + (hy * (hx * a[2 * k] + lx * b[2 * k]) + ly * (hx * c[2 * k] + lx * d[2 * k]));
    const float r1 = v[2 * k + 1] + (hy * (hx * a[2 * k + 1] + lx * b[2 * k + 1]) + ly * (hx * c[2 * k + 1] + lx * d[2 * k + 1]));
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(ow[k]) : "f"(r1), "f"(r0));
  }
  *reinterpret_cast<uint4*>(static_cast<unsigned short*>(dst) + de) = o;
}

// fp32 [rows][cin] -> bf16 [rows][cin_pad] (zero padded): conv weights for the bf16 tensor-core path
__global__ void weights_to_bf16_kernel(const float* __restrict__ src, unsigned short* __restrict__ dst, size_t rows,
                                       int cin, int cin_pad) {
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= rows * cin_pad) return;
  const size_t r = idx / cin_pad;
  const int c = static_cast<int>(idx % cin_pad);
  dst[idx] = c < cin ? f2bf(src[r * cin + c]) : static_cast<unsigned short>(0);
}

// ------------------------------------------------------------------------------------------ posenc
__global__ void posenc_kernel(const float* __restrict__ feat, const float* __restrict__ pe,
                              float* __restrict__ tok, long long ldt, int N, int L, int C4) {
  const size_t total = static_cast<size_t>(N) * L * C4;
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c4 = static_cast<int>(idx % C4);
  const size_t row = idx / C4;
  const int l = static_cast<int>(row % L);
  const float4 f = reinterpret_cast<const float4*>(feat)[idx];
  const float4 p = reinterpret_cast<const float4*>(pe)[static_cast<size_t>(l) * C4 + c4];
  float4 o;
  o.x = f.x + p.x; o.y = f.y + p.y; o.z = f.z + p.z; o.w = f.w + p.w;
  *reinterpret_cast<float4*>(tok + row * ldt + c4 * 4) = o;
}

// ------------------------------------------------------------------------------------------ linear attention (long)
// 8 heads x 32 (coarse level). One warp = one head; lane = value column v.
//   kv_partial : block (8 warps) reduces a slab of tokens for all heads. K rows are staged in shared
//                memory (broadcast reads), V is read straight into registers (coalesced).
//   kv_reduce  : sums the slabs.
//   attn_apply : each lane keeps KV[h][:, v] and Ksum[h][lane] in registers; q rows are broadcast
//                from shared memory; one warp-shuffle reduction per token for the normaliser.
// Both streaming kernels move their token rows with a 3-stage cp.async pipeline (16 tokens x 1 KB per
// operand per stage), so the HBM latency is paid once per block, not once per slab.
constexpr int kSlab = 16;     // tokens per pipeline stage
constexpr int kAttStages = 3;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  const int sz = valid ? 16 : 0;   // src-size 0 => the 16 bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// rows [r0, r0+kSlab) of an fp32 [rows][256] matrix (row stride ld floats) -> dst[kSlab][256];
// rows >= r_end are zero-filled
__device__ __forceinline__ void slab_load(void* dst, const void* __restrict__ src, long long ld, long long r0,
                                          long long r_end, int t) {
  constexpr int kChunks = 64;                       // 16-byte chunks per row
#pragma unroll
  for (int i = 0; i < kSlab * kChunks / 256; ++i) {
    const int c = t + 256 * i;
    const int r = c / kChunks, ch = c % kChunks;
    const bool ok = r0 + r < r_end;
    cp_async16(static_cast<char*>(dst) + (r * kChunks + ch) * 16,
               static_cast<const char*>(src) + ((ok ? (r0 + r) : r0) * ld) * 4 + ch * 16, ok);
  }
}
// element t of row r / the 32 channels of head h of row r, from a staged slab
__device__ __forceinline__ float slab_elem(const void* slab, int r, int t) {
  return static_cast<const float*>(slab)[r * 256 + t];
}
__device__ __forceinline__ void slab_head(const void* slab, int r, int h, float (&o)[32]) {
  const float4* p = reinterpret_cast<const float4*>(static_cast<const float*>(slab) + r * 256 + h * 32);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 f = p[q];
    o[4 * q] = f.x; o[4 * q + 1] = f.y; o[4 * q + 2] = f.z; o[4 * q + 3] = f.w;
  }
}

__global__ void __launch_bounds__(256) kv_partial_kernel(const void* __restrict__ K, long long ldk,
                                                         const void* __restrict__ V, long long ldv,
                                                         float* __restrict__ kv_part, int S, int splits) {
  extern __shared__ __align__(16) float att_smem[];
  constexpr int kSlabBytes = kSlab * 256 * 4;
  char* sK = reinterpret_cast<char*>(att_smem);                          // [stages][kSlab][256]
  char* sV = reinterpret_cast<char*>(att_smem) + kAttStages * kSlabBytes;
  const int split = blockIdx.x, n = blockIdx.y;
  const int chunk = (S + splits - 1) / splits;
  const int s_beg = split * chunk, s_end = min(S, s_beg + chunk);
  const int t = threadIdx.x, h = t >> 5, lane = t & 31;
  const long long base = static_cast<long long>(n) * S;
  const int nslab = s_end > s_beg ? (s_end - s_beg + kSlab - 1) / kSlab : 0;
  float acc[32];
#pragma unroll
  for (int d = 0; d < 32; ++d) acc[d] = 0.f;
  float ks = 0.f;
  const float fS = static_cast<float>(S);
#pragma unroll
  for (int st = 0; st < kAttStages - 1; ++st) {
    if (st < nslab) {
      slab_load(sK + st * kSlabBytes, K, ldk, base + s_beg + st * kSlab, base + s_end, t);
      slab_load(sV + st * kSlabBytes, V, ldv, base + s_beg + st * kSlab, base + s_end, t);
    }
    cp_async_commit();
  }
  for (int i = 0; i < nslab; ++i) {
    cp_async_wait<kAttStages - 2>();
    __syncthreads();   // slab i has landed for everyone; everyone is done with slab i-1 (its stage is refilled now)
    {
      const int nx = i + kAttStages - 1;
      if (nx < nslab) {
        const int st = nx % kAttStages;
        slab_load(sK + st * kSlabBytes, K, ldk, base + s_beg + nx * kSlab, base + s_end, t);
        slab_load(sV + st * kSlabBytes, V, ldv, base + s_beg + nx * kSlab, base + s_end, t);
      }
      cp_async_commit();
    }
    const char* k0 = sK + (i % kAttStages) * kSlabBytes;
    const char* v0 = sV + (i % kAttStages) * kSlabBytes;
#pragma unroll 4
    for (int r = 0; r < kSlab; ++r) {
      const float vv = __fdiv_rn(slab_elem(v0, r, t), fS);     // values / v_length (linear_attention.py:40)
      float kk[32];
      slab_head(k0, r, h, kk);
#pragma unroll
      for (int d = 0; d < 32; ++d) acc[d] = fmaf(kk[d], vv, acc[d]);
      ks += slab_elem(k0, r, t);
    }
  }
  float* o = kv_part + ((static_cast<size_t>(n) * splits + split) * 8 + h) * 1056;
#pragma unroll
  for (int d = 0; d < 32; ++d) o[d * 32 + lane] = acc[d];
  o[1024 + lane] = ks;
}

__global__ void __launch_bounds__(256) kv_reduce_kernel(const float* __restrict__ kv_part,
                                                        float* __restrict__ kv, int splits) {
  // grid (ceil(8448/256), n): element e of the [8][1056] block of image n
  const int n = blockIdx.y;
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= 8 * 1056) return;
  float s = 0.f;
  for (int k = 0; k < splits; ++k) s += kv_part[(static_cast<size_t>(n) * splits + k) * 8448 + e];
  kv[static_cast<size_t>(n) * 8448 + e] = s;
}

__global__ void __launch_bounds__(256) attn_apply_kernel(const void* __restrict__ Q, long long ldq,
                                                         const float* __restrict__ kv,
                                                         void* __restrict__ msg, long long ldm, int L,
                                                         int S, float eps, int splits) {
  extern __shared__ __align__(16) float att_smem[];
  constexpr int kSlabBytes = kSlab * 256 * 4;
  char* sQ = reinterpret_cast<char*>(att_smem);                           // [stages][kSlab][256]
  const int n = blockIdx.y;
  const int chunk = (L + splits - 1) / splits;
  const int l_beg = blockIdx.x * chunk, l_end = min(L, l_beg + chunk);
  const int nslab = l_end > l_beg ? (l_end - l_beg + kSlab - 1) / kSlab : 0;
  const int t = threadIdx.x, h = t >> 5, lane = t & 31;
  const long long base = static_cast<long long>(n) * L;
#pragma unroll
  for (int st = 0; st < kAttStages - 1; ++st) {
    if (st < nslab) slab_load(sQ + st * kSlabBytes, Q, ldq, base + l_beg + st * kSlab, base + l_end, t);
    cp_async_commit();
  }
  const float* kvh = kv + (static_cast<size_t>(n) * 8 + h) * 1056;
  float kvr[32];
#pragma unroll
  for (int d = 0; d < 32; ++d) kvr[d] = kvh[d * 32 + lane];
  const float ksum = kvh[1024 + lane];
  const float fS = static_cast<float>(S);
  for (int i = 0; i < nslab; ++i) {
    cp_async_wait<kAttStages - 2>();
    __syncthreads();
    {
      const int nx = i + kAttStages - 1;
      if (nx < nslab) slab_load(sQ + (nx % kAttStages) * kSlabBytes, Q, ldq, base + l_beg + nx * kSlab, base + l_end, t);
      cp_async_commit();
    }
    const char* q0 = sQ + (i % kAttStages) * kSlabBytes;
    const int cnt = min(kSlab, l_end - l_beg - i * kSlab);
#pragma unroll 4
    for (int r = 0; r < cnt; ++r) {
      float qq[32];
      slab_head(q0, r, h, qq);
      float a = 0.f;
#pragma unroll
      for (int d = 0; d < 32; ++d) a = fmaf(qq[d], kvr[d], a);
      const float den = warp_sum(slab_elem(q0, r, t) * ksum);
      const float o = a * (1.f / (den + eps)) * fS;
      const long long oi = (base + l_beg + i * kSlab + r) * ldm + t;
      static_cast<float*>(msg)[oi] = o;
    }
  }
}


// ------------------------------------------------------------------------------------------ linear attention on mma.sync (bf16 operands)
// bf16 mode: q, k and v are bf16 in HBM, so K'^T V (32 x 32 per head, reduction over the tokens) and Q' (KV) are
// warp-level m16n8k16 tensor-core products with fp32 accumulation; SIMT kernels like the fp32 ones above would be
// issue-bound on shared-memory reads and fp32 FMAs. Slabs land by cp.async with the 16-byte chunk index XOR-ed by
// (row & 7), which makes every ldmatrix phase (8 rows, one chunk column) bank-conflict free. The reference's
// values / v_length ... * v_length pair (linear_attention.py:40-45) cancels and is not applied here.
constexpr int kMS = 32;          // tokens per pipeline stage
constexpr int kMStages = 3;
constexpr int kMSlabBytes = kMS * 512;

__device__ __forceinline__ void ldsm_x4(unsigned (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(static_cast<unsigned>(__cvta_generic_to_shared(p))));
}
__device__ __forceinline__ void ldsm_x4_t(unsigned (&r)[4], const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(static_cast<unsigned>(__cvta_generic_to_shared(p))));
}
__device__ __forceinline__ void mma_bf16(float (&c)[4], const unsigned (&a)[4], unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ unsigned pack_bf16(float lo, float hi) {
  return static_cast<unsigned>(f2bf(lo)) | (static_cast<unsigned>(f2bf(hi)) << 16);
}
// rows [r0, r0+kMS) of a bf16 [rows][256] matrix -> dst[kMS][512 B], chunk-swizzled; rows >= r_end are zero-filled
__device__ __forceinline__ void slab_load_sw(char* dst, const void* __restrict__ src, long long ld, long long r0,
                                             long long r_end, int t) {
#pragma unroll
  for (int i = 0; i < kMS * 32 / 256; ++i) {
    const int c = t + 256 * i;
    const int r = c >> 5, ch = c & 31;
    const bool ok = r0 + r < r_end;
    cp_async16(dst + r * 512 + ((ch ^ (r & 7)) << 4),
               static_cast<const char*>(src) + ((ok ? (r0 + r) : r0) * ld) * 2 + ch * 16, ok);
  }
}
__device__ __forceinline__ const char* sw_addr(const char* slab, int row, int chunk) {
  return slab + row * 512 + ((chunk ^ (row & 7)) << 4);
}

// kv_part[n][split][h][d*32 + v] = sum_s K'[s][32h+d] V[s][32h+v],  [..][1024 + d] = sum_s K'[s][32h+d]; warp = head
__device__ __forceinline__ float elu1_fast(float v) {   // the token-GEMM epilogue's elu(x) + 1 (conv_gemm.cu act_fn<ACT_ELU1, true>)
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fminf(v * 1.4426950408889634f, 0.f)));
  return fmaxf(v, 0.f) + e;
}
// The bf16 attention kernels take q and k as the projection GEMM leaves them and apply the feature map
// elu(x) + 1 to the mma fragments in registers: the GEMM's 8 epilogue warps were bound by exactly this (MUFU + ALU issue),
// while these kernels wait for HBM. keep_lo / keep_hi = false zeroes an element (token padding: K' rows past the end).
__device__ __forceinline__ unsigned elu1_bf16x2(unsigned v, bool keep_lo = true, bool keep_hi = true) {
  const float lo = elu1_fast(__uint_as_float(v << 16)), hi = elu1_fast(__uint_as_float(v & 0xffff0000u));
  return pack_bf16(keep_lo ? lo : 0.f, keep_hi ? hi : 0.f);
}

__global__ void __launch_bounds__(256) kv_partial_mma_kernel(const void* __restrict__ K, long long ldk,
                                                             const void* __restrict__ V, long long ldv,
                                                             float* __restrict__ kv_part, int S, int splits) {
  extern __shared__ __align__(128) float att_smem[];
  char* sK = reinterpret_cast<char*>(att_smem);
  char* sV = sK + kMStages * kMSlabBytes;
  const int split = blockIdx.x, n = blockIdx.y;
  const int chunk = (S + splits - 1) / splits;
  const int s_beg = split * chunk, s_end = min(S, s_beg + chunk);
  const int t = threadIdx.x, h = t >> 5, lane = t & 31;
  const int j = lane >> 3, r = lane & 7, g = lane >> 2, tq = lane & 3;
  const long long base = static_cast<long long>(n) * S;
  const int nslab = s_end > s_beg ? (s_end - s_beg + kMS - 1) / kMS : 0;
  float acc[2][4][4], accs[2][4];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      accs[a][b] = 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
    }
  }
  const unsigned ones = (g == 0) ? 0x3F803F80u : 0u;      // B tile whose column 0 is all ones -> sum of K' over the tokens
#pragma unroll
  for (int st = 0; st < kMStages - 1; ++st) {
    if (st < nslab) {
      slab_load_sw(sK + st * kMSlabBytes, K, ldk, base + s_beg + st * kMS, base + s_end, t);
      slab_load_sw(sV + st * kMSlabBytes, V, ldv, base + s_beg + st * kMS, base + s_end, t);
    }
    cp_async_commit();
  }
  for (int i = 0; i < nslab; ++i) {
    cp_async_wait<kMStages - 2>();
    __syncthreads();
    {
      const int nx = i + kMStages - 1;
      if (nx < nslab) {
        const int st = nx % kMStages;
        slab_load_sw(sK + st * kMSlabBytes, K, ldk, base + s_beg + nx * kMS, base + s_end, t);
        slab_load_sw(sV + st * kMSlabBytes, V, ldv, base + s_beg + nx * kMS, base + s_end, t);
      }
      cp_async_commit();
    }
    const char* k0 = sK + (i % kMStages) * kMSlabBytes;
    const char* v0 = sV + (i % kMStages) * kMSlabBytes;
#pragma unroll
    for (int ks = 0; ks < kMS / 16; ++ks) {
      unsigned a[2][4], b[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)      // A = K'^T: m = channel d, k = token
        ldsm_x4_t(a[mt], sw_addr(k0, 16 * ks + r + 8 * (j >> 1), 4 * h + 2 * mt + (j & 1)));
      // registers e = 0, 1 hold tokens 2 tq, 2 tq + 1 of the k-step, e = 2, 3 those + 8
      const int tok = s_beg + i * kMS + 16 * ks + 2 * tq;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int t0 = tok + 8 * (e >> 1);
          a[mt][e] = elu1_bf16x2(a[mt][e], t0 < s_end, t0 + 1 < s_end);
        }
#pragma unroll
      for (int pp = 0; pp < 2; ++pp)      // B = V: k = token, n = channel v (two 8-wide tiles per ldmatrix)
        ldsm_x4_t(b[pp], sw_addr(v0, 16 * ks + r + 8 * (j & 1), 4 * h + 2 * pp + (j >> 1)));
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma_bf16(acc[mt][nt], a[mt], b[nt >> 1][2 * (nt & 1)], b[nt >> 1][2 * (nt & 1) + 1]);
        mma_bf16(accs[mt], a[mt], ones, ones);
      }
    }
  }
  float* o = kv_part + ((static_cast<size_t>(n) * splits + split) * 8 + h) * 1056;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      *reinterpret_cast<float2*>(o + (16 * mt + g) * 32 + 8 * nt + 2 * tq) = make_float2(acc[mt][nt][0], acc[mt][nt][1]);
      *reinterpret_cast<float2*>(o + (16 * mt + g + 8) * 32 + 8 * nt + 2 * tq) = make_float2(acc[mt][nt][2], acc[mt][nt][3]);
    }
    if (tq == 0) {
      o[1024 + 16 * mt + g] = accs[mt][0];
      o[1024 + 16 * mt + g + 8] = accs[mt][2];
    }
  }
}

// msg[l][32h+v] = (Q'[l] . KV[:, v]) / (Q'[l] . Ksum + eps), KV / Ksum rounded to bf16 as the B operand; warp = head
__global__ void __launch_bounds__(256) attn_apply_mma_kernel(const void* __restrict__ Q, long long ldq,
                                                             const float* __restrict__ kv,
                                                             unsigned short* __restrict__ msg, long long ldm, int L,
                                                             float eps, int splits) {
  extern __shared__ __align__(128) float att_smem[];
  char* sQ = reinterpret_cast<char*>(att_smem);
  const int n = blockIdx.y;
  const int chunk = (L + splits - 1) / splits;
  const int l_beg = blockIdx.x * chunk, l_end = min(L, l_beg + chunk);
  const int nslab = l_end > l_beg ? (l_end - l_beg + kMS - 1) / kMS : 0;
  const int t = threadIdx.x, h = t >> 5, lane = t & 31;
  const int j = lane >> 3, r = lane & 7, g = lane >> 2, tq = lane & 3;
  const long long base = static_cast<long long>(n) * L;
#pragma unroll
  for (int st = 0; st < kMStages - 1; ++st) {
    if (st < nslab) slab_load_sw(sQ + st * kMSlabBytes, Q, ldq, base + l_beg + st * kMS, base + l_end, t);
    cp_async_commit();
  }
  const float* kvh = kv + (static_cast<size_t>(n) * 8 + h) * 1056;
  unsigned bkv[2][4][2], bden[2][2];      // B fragments: k = channel d (two 16-steps), n = channel v (four tiles) / the Ksum column
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    const int d0 = 16 * ks + 2 * tq;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int v = 8 * nt + g;
      bkv[ks][nt][0] = pack_bf16(kvh[d0 * 32 + v], kvh[(d0 + 1) * 32 + v]);
      bkv[ks][nt][1] = pack_bf16(kvh[(d0 + 8) * 32 + v], kvh[(d0 + 9) * 32 + v]);
    }
    bden[ks][0] = g == 0 ? pack_bf16(kvh[1024 + d0], kvh[1024 + d0 + 1]) : 0u;
    bden[ks][1] = g == 0 ? pack_bf16(kvh[1024 + d0 + 8], kvh[1024 + d0 + 9]) : 0u;
  }
  for (int i = 0; i < nslab; ++i) {
    cp_async_wait<kMStages - 2>();
    __syncthreads();
    {
      const int nx = i + kMStages - 1;
      if (nx < nslab) slab_load_sw(sQ + (nx % kMStages) * kMSlabBytes, Q, ldq, base + l_beg + nx * kMS, base + l_end, t);
      cp_async_commit();
    }
    const char* q0 = sQ + (i % kMStages) * kMSlabBytes;
#pragma unroll
    for (int mt = 0; mt < kMS / 16; ++mt) {
      float c[4][4], cd[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        cd[b] = 0.f;
#pragma unroll
        for (int e = 0; e < 4; ++e) c[b][e] = 0.f;
      }
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        unsigned a[4];                      // A = Q': m = token, k = channel d
        ldsm_x4(a, sw_addr(q0, 16 * mt + r + 8 * (j & 1), 4 * h + 2 * ks + (j >> 1)));
#pragma unroll
        for (int e = 0; e < 4; ++e) a[e] = elu1_bf16x2(a[e]);
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma_bf16(c[nt], a, bkv[ks][nt][0], bkv[ks][nt][1]);
        mma_bf16(cd, a, bden[ks][0], bden[ks][1]);
      }
      const float den_lo = __shfl_sync(0xffffffffu, cd[0], lane & ~3), den_hi = __shfl_sync(0xffffffffu, cd[2], lane & ~3);
      const float z_lo = 1.f / (den_lo + eps), z_hi = 1.f / (den_hi + eps);
      const int l0 = l_beg + i * kMS + 16 * mt + g;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        if (l0 < l_end)
          *reinterpret_cast<unsigned*>(msg + (base + l0) * ldm + 32 * h + 8 * nt + 2 * tq) = pack_bf16(c[nt][0] * z_lo, c[nt][1] * z_lo);
        if (l0 + 8 < l_end)
          *reinterpret_cast<unsigned*>(msg + (base + l0 + 8) * ldm + 32 * h + 8 * nt + 2 * tq) = pack_bf16(c[nt][2] * z_hi, c[nt][3] * z_hi);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------ linear attention (windows)
// C = 128 (8 heads x 16), T tokens per item (T <= 32). One block (128 threads) per item.
template <int T>
__global__ void __launch_bounds__(128) attn_windows_kernel(const void* __restrict__ Qv, long long ldq,
                                                           const void* __restrict__ Kv, long long ldk,
                                                           const void* __restrict__ Vv, long long ldv,
                                                           void* __restrict__ msgv, long long ldm,
                                                           const int* __restrict__ n_items_dev,
                                                           float eps) {
  const int item = blockIdx.x;
  if (item >= *n_items_dev) return;
  __shared__ __align__(16) float sQ[T][128];
  __shared__ __align__(16) float sK[T][128];   // K rows, later the output rows
  __shared__ __align__(16) float sV[T][128];
  const int t = threadIdx.x;
  const int hb = (t >> 4) << 4;  // first channel of this thread's head
  const float fT = static_cast<float>(T);
  // cooperative 16-byte loads of the item's T x 128 q / k / v rows
  constexpr int CH = 32, EPC = 4;     // chunks per row, elements per chunk
  const size_t row0 = static_cast<size_t>(item) * T;
  for (int c = t; c < T * CH; c += 128) {
    const int r = c / CH, e0 = (c % CH) * EPC;
    float q[EPC], k[EPC], v[EPC];
    const float4 fq = *reinterpret_cast<const float4*>(static_cast<const float*>(Qv) + (row0 + r) * ldq + e0);
    const float4 fk = *reinterpret_cast<const float4*>(static_cast<const float*>(Kv) + (row0 + r) * ldk + e0);
    const float4 fv = *reinterpret_cast<const float4*>(static_cast<const float*>(Vv) + (row0 + r) * ldv + e0);
    q[0] = fq.x; q[1] = fq.y; q[2] = fq.z; q[3] = fq.w;
    k[0] = fk.x; k[1] = fk.y; k[2] = fk.z; k[3] = fk.w;
    v[0] = fv.x; v[1] = fv.y; v[2] = fv.z; v[3] = fv.w;
#pragma unroll
    for (int e = 0; e < EPC; e += 4) {                 // 16-byte shared-memory stores
      *reinterpret_cast<float4*>(&sQ[r][e0 + e]) = make_float4(q[e], q[e + 1], q[e + 2], q[e + 3]);
      *reinterpret_cast<float4*>(&sK[r][e0 + e]) = make_float4(k[e], k[e + 1], k[e + 2], k[e + 3]);
      *reinterpret_cast<float4*>(&sV[r][e0 + e]) =     // values / v_length (linear_attention.py:40)
          make_float4(__fdiv_rn(v[e], fT), __fdiv_rn(v[e + 1], fT), __fdiv_rn(v[e + 2], fT), __fdiv_rn(v[e + 3], fT));
    }
  }
  __syncthreads();
  float kvc[16], ks[16];
#pragma unroll
  for (int d = 0; d < 16; ++d) { kvc[d] = 0.f; ks[d] = 0.f; }
#pragma unroll
  for (int s = 0; s < T; ++s) {
    const float vs = sV[s][t];
    const float4* kr = reinterpret_cast<const float4*>(&sK[s][hb]);
#pragma unroll
    for (int d4 = 0; d4 < 4; ++d4) {
      const float4 kk = kr[d4];
      kvc[4 * d4] = fmaf(kk.x, vs, kvc[4 * d4]);         ks[4 * d4] += kk.x;
      kvc[4 * d4 + 1] = fmaf(kk.y, vs, kvc[4 * d4 + 1]); ks[4 * d4 + 1] += kk.y;
      kvc[4 * d4 + 2] = fmaf(kk.z, vs, kvc[4 * d4 + 2]); ks[4 * d4 + 2] += kk.z;
      kvc[4 * d4 + 3] = fmaf(kk.w, vs, kvc[4 * d4 + 3]); ks[4 * d4 + 3] += kk.w;
    }
  }
  __syncthreads();                                     // everyone is done with sK: it now collects the output rows
#pragma unroll 5
  for (int l = 0; l < T; ++l) {
    const float4* qr = reinterpret_cast<const float4*>(&sQ[l][hb]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int d4 = 0; d4 < 4; ++d4) {
      const float4 q = qr[d4];
      num = fmaf(q.x, kvc[4 * d4], num);     den = fmaf(q.x, ks[4 * d4], den);
      num = fmaf(q.y, kvc[4 * d4 + 1], num); den = fmaf(q.y, ks[4 * d4 + 1], den);
      num = fmaf(q.z, kvc[4 * d4 + 2], num); den = fmaf(q.z, ks[4 * d4 + 2], den);
      num = fmaf(q.w, kvc[4 * d4 + 3], num); den = fmaf(q.w, ks[4 * d4 + 3], den);
    }
    sK[l][t] = num * (1.f / (den + eps)) * fT;
  }
  __syncthreads();
  for (int c = t; c < T * CH; c += 128) {              // 16-byte stores of the T x 128 message rows
    const int r = c / CH, e0 = (c % CH) * EPC;
    *reinterpret_cast<float4*>(static_cast<float*>(msgv) + (row0 + r) * ldm + e0) =
        make_float4(sK[r][e0], sK[r][e0 + 1], sK[r][e0 + 2], sK[r][e0 + 3]);
  }
}


// bf16 variant on mma.sync: block = window (8 warps = 8 heads of 16 channels), tokens padded 25 -> 32 with zero K' / V
// rows. Per head: KV^T[v][d] = sum_s V[s][v] K'[s][d] (A = V^T, B = K') and Ksum through an A tile whose row 0 is all
// ones; the accumulator fragments ARE the B fragments of the second product out[l][v] = Q'[l][d] KV[d][v] (transposed
// accumulation puts (d pair, v) in the right lanes), so nothing goes back through shared memory.
template <int T>
__global__ void __launch_bounds__(256) attn_windows_mma_kernel(const unsigned short* __restrict__ Q, long long ldq,
                                                               const unsigned short* __restrict__ K, long long ldk,
                                                               const unsigned short* __restrict__ V, long long ldv,
                                                               unsigned short* __restrict__ msg, long long ldm,
                                                               const int* __restrict__ n_items_dev, float eps) {
  static_assert(T <= 32, "window tokens are padded to 32");
  const int item = blockIdx.x;
  if (item >= *n_items_dev) return;
  __shared__ __align__(128) char sm[3][32 * 256];        // Q', K', V: [32 rows][128 ch] bf16, 16-byte chunks XOR (row & 7)
  const int t = threadIdx.x;
  const size_t row0 = static_cast<size_t>(item) * T;
  for (int c = t; c < 3 * T * 16; c += 256) {
    const int which = c / (T * 16), rc = c % (T * 16), r = rc >> 4, ch = rc & 15;
    const unsigned short* src = which == 0 ? Q + (row0 + r) * ldq : which == 1 ? K + (row0 + r) * ldk : V + (row0 + r) * ldv;
    cp_async16(sm[which] + r * 256 + ((ch ^ (r & 7)) << 4), src + ch * 8, true);
  }
  cp_async_commit();
  for (int c = t; c < 2 * (32 - T) * 16; c += 256) {     // zero padding rows of K' and V
    const int which = 1 + c / ((32 - T) * 16), rc = c % ((32 - T) * 16), r = T + (rc >> 4), ch = rc & 15;
    *reinterpret_cast<uint4*>(sm[which] + r * 256 + (ch << 4)) = make_uint4(0, 0, 0, 0);
  }
  cp_async_wait<0>();
  __syncthreads();
  const int h = t >> 5, lane = t & 31;
  const int j = lane >> 3, r = lane & 7, g = lane >> 2, tq = lane & 3;
  auto addr = [&](int which, int row, int chunk) { return sm[which] + row * 256 + ((chunk ^ (row & 7)) << 4); };
  float ckv[2][4], cks[2][4];                            // [d tile]: KV^T rows v = g / g+8, cols d = 8 j' + 2 tq (+1)
#pragma unroll
  for (int a = 0; a < 2; ++a) {
#pragma unroll
    for (int e = 0; e < 4; ++e) { ckv[a][e] = 0.f; cks[a][e] = 0.f; }
  }
  const unsigned one = (g == 0) ? 0x3F803F80u : 0u;
  const unsigned aones[4] = {one, 0u, one, 0u};
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    unsigned a[4], b[4];
    ldsm_x4_t(a, addr(2, 16 * ks + r + 8 * (j >> 1), 2 * h + (j & 1)));     // A = V^T: m = v, k = token
    ldsm_x4_t(b, addr(1, 16 * ks + r + 8 * (j & 1), 2 * h + (j >> 1)));     // B = K': k = token, n = d
    // b[2 nt] holds tokens 2 tq, 2 tq + 1 of the k-step, b[2 nt + 1] those + 8; rows >= T stay zero
    const int tok = 16 * ks + 2 * tq;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int t0 = tok + 8 * (e & 1);
      b[e] = elu1_bf16x2(b[e], t0 < T, t0 + 1 < T);
    }
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      mma_bf16(ckv[nt], a, b[2 * nt], b[2 * nt + 1]);
      mma_bf16(cks[nt], aones, b[2 * nt], b[2 * nt + 1]);
    }
  }
  const unsigned bv0[2] = {pack_bf16(ckv[0][0], ckv[0][1]), pack_bf16(ckv[1][0], ckv[1][1])};   // n tile v 0-7
  const unsigned bv1[2] = {pack_bf16(ckv[0][2], ckv[0][3]), pack_bf16(ckv[1][2], ckv[1][3])};   // n tile v 8-15
  const unsigned bd[2] = {pack_bf16(cks[0][0], cks[0][1]), pack_bf16(cks[1][0], cks[1][1])};    // column 0 = Ksum
#pragma unroll
  for (int mt = 0; mt < 2; ++mt) {
    unsigned a[4];
    ldsm_x4(a, addr(0, 16 * mt + r + 8 * (j & 1), 2 * h + (j >> 1)));       // A = Q': m = token, k = d
#pragma unroll
    for (int e = 0; e < 4; ++e) a[e] = elu1_bf16x2(a[e]);
    float c0[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f}, cd[4] = {0.f, 0.f, 0.f, 0.f};
    mma_bf16(c0, a, bv0[0], bv0[1]);
    mma_bf16(c1, a, bv1[0], bv1[1]);
    mma_bf16(cd, a, bd[0], bd[1]);
    const float den_lo = __shfl_sync(0xffffffffu, cd[0], lane & ~3), den_hi = __shfl_sync(0xffffffffu, cd[2], lane & ~3);
    const float z_lo = 1.f / (den_lo + eps), z_hi = 1.f / (den_hi + eps);
    const int l0 = 16 * mt + g;
    if (l0 < T) {
      unsigned short* o = msg + (row0 + l0) * ldm + 16 * h + 2 * tq;
      *reinterpret_cast<unsigned*>(o) = pack_bf16(c0[0] * z_lo, c0[1] * z_lo);
      *reinterpret_cast<unsigned*>(o + 8) = pack_bf16(c1[0] * z_lo, c1[1] * z_lo);
    }
    if (l0 + 8 < T) {
      unsigned short* o = msg + (row0 + l0 + 8) * ldm + 16 * h + 2 * tq;
      *reinterpret_cast<unsigned*>(o) = pack_bf16(c0[2] * z_hi, c0[3] * z_hi);
      *reinterpret_cast<unsigned*>(o + 8) = pack_bf16(c1[2] * z_hi, c1[3] * z_hi);
    }
  }
}

// ------------------------------------------------------------------------------------------ layernorm
template <int C>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ in, long long ldi,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta,
                                                        const float* __restrict__ res, long long ldr,
                                                        float* __restrict__ out, long long ldo,
                                                        long long rows, const int* __restrict__ dyn_rows) {
  constexpr int V = C / 128;  // float4 per lane
  long long lim = rows;
  if (dyn_rows) lim = min(lim, static_cast<long long>(*dyn_rows));
  const int lane = threadIdx.x & 31;
  for (long long row = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5); row < lim;
       row += static_cast<long long>(gridDim.x) * 8) {
  float x[4 * V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const float4 f = *reinterpret_cast<const float4*>(in + row * ldi + k * 128 + lane * 4);
    x[4 * k] = f.x; x[4 * k + 1] = f.y; x[4 * k + 2] = f.z; x[4 * k + 3] = f.w;
  }
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 4 * V; ++k) s += x[k];
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int k = 0; k < 4 * V; ++k) {
    const float d = x[k] - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = 1.f / sqrtf(warp_sum(q) / C + 1e-5f);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    const int c = k * 128 + lane * 4;
    const float4 g = *reinterpret_cast<const float4*>(gamma + c);
    const float4 b = *reinterpret_cast<const float4*>(beta + c);
    float4 o;
    o.x = (x[4 * k] - mean) * rstd * g.x + b.x;
    o.y = (x[4 * k + 1] - mean) * rstd * g.y + b.y;
    o.z = (x[4 * k + 2] - mean) * rstd * g.z + b.z;
    o.w = (x[4 * k + 3] - mean) * rstd * g.w + b.w;
    if (res) {
      const float4 r = *reinterpret_cast<const float4*>(res + row * ldr + c);
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    *reinterpret_cast<float4*>(out + row * ldo + c) = o;
  }
  }
}

// dst16[row][0..C) = bf16(src[row][0..C)), 4 channels per thread
__global__ void rows_to_bf16_kernel(const float* __restrict__ src, long long lds, unsigned short* __restrict__ dst,
                                    long long ldd, long long rows, int C4, const int* __restrict__ dyn_rows) {
  long long lim = rows;
  if (dyn_rows) lim = min(lim, static_cast<long long>(*dyn_rows));
  const long long total = lim * C4;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / C4;
    const int c = static_cast<int>(i - row * C4) * 4;
    const float4 f = *reinterpret_cast<const float4*>(src + row * lds + c);
    uint2 u;
    u.x = static_cast<unsigned>(f2bf(f.x)) | (static_cast<unsigned>(f2bf(f.y)) << 16);
    u.y = static_cast<unsigned>(f2bf(f.z)) | (static_cast<unsigned>(f2bf(f.w)) << 16);
    *reinterpret_cast<uint2*>(dst + row * ldd + c) = u;
  }
}

// fp32-faithful GEMM operands (precision mode 2, "3xTF32"): x = hi + lo with hi = tf32(x), lo = tf32(x - hi), so that
//   A.B ~= Ahi.Bhi + Alo.Bhi + Ahi.Blo   (the dropped lo.lo term and the rounding of lo are ~2^-22 relative)
// is ONE tensor-core GEMM over a three times longer K: dst row = [hi | lo | hi] (pattern 0, the A operand) or
// [hi | hi | lo] (pattern 1, the B operand). Both halves are exact TF32 values, so the tensor core's own
// fp32 -> tf32 conversion of the operands is the identity.
__device__ __forceinline__ float tf32_rn(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__global__ void rows_split3_kernel(const float* __restrict__ src, long long lds, long long src_img_stride,
                                   float* __restrict__ dst, long long rows_per_img, int C4, int pattern,
                                   const int* __restrict__ dyn_rows) {
  long long lim = rows_per_img;
  if (dyn_rows) lim = min(lim, static_cast<long long>(*dyn_rows));
  const int img = blockIdx.y;
  const long long total = lim * C4;
  const int C = C4 * 4;
  const float* s = src + img * src_img_stride;
  float* d0 = dst + img * rows_per_img * 3 * C;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / C4;
    const int c = static_cast<int>(i - row * C4) * 4;
    const float4 f = *reinterpret_cast<const float4*>(s + row * lds + c);
    float4 hi, lo;
    hi.x = tf32_rn(f.x); hi.y = tf32_rn(f.y); hi.z = tf32_rn(f.z); hi.w = tf32_rn(f.w);
    lo.x = tf32_rn(f.x - hi.x); lo.y = tf32_rn(f.y - hi.y); lo.z = tf32_rn(f.z - hi.z); lo.w = tf32_rn(f.w - hi.w);
    float* d = d0 + row * 3 * C + c;
    *reinterpret_cast<float4*>(d) = hi;
    *reinterpret_cast<float4*>(d + C) = pattern == 0 ? lo : hi;
    *reinterpret_cast<float4*>(d + 2 * C) = pattern == 0 ? hi : lo;
  }
}

// ------------------------------------------------------------------------------------------ coarse matching
// conf = softmax_col(S) * softmax_row(S); the expression is written with explicit rounding
// intrinsics so that every pass reproduces the identical fp32 value (the mutual-NN test compares
// for float equality, coarse_matching.py:187-189).
__device__ __forceinline__ float conf_value(float s, float rmax, float rrs, float cmax, float crs,
                                            bool raw = false) {
  if (raw) return s;  // the input already is the confidence matrix (stage-boundary entry point)
  const float pr = __fmul_rn(__expf(__fsub_rn(s, rmax)), rrs);
  const float pc = __fmul_rn(__expf(__fsub_rn(s, cmax)), crs);
  return __fmul_rn(pc, pr);
}

__device__ __forceinline__ float block_max_256(float v, float* sh) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = sh[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) r = fmaxf(r, sh[k]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_sum_256(float v, float* sh) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) r += sh[k];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(256) row_stats_kernel(const float* __restrict__ S,
                                                        float* __restrict__ row_max,
                                                        float* __restrict__ row_rsum, int L) {
  __shared__ float sh[8];
  const size_t r = static_cast<size_t>(blockIdx.y) * L + blockIdx.x;
  const float* p = S + r * L;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < L; j += 256) m = fmaxf(m, p[j]);
  m = block_max_256(m, sh);
  float s = 0.f;
  for (int j = threadIdx.x; j < L; j += 256) s += __expf(__fsub_rn(p[j], m));
  s = block_sum_256(s, sh);
  if (threadIdx.x == 0) {
    row_max[r] = m;
    row_rsum[r] = 1.f / s;
  }
}

// column stats: partial online (max, sum) over a slab of rows
__global__ void __launch_bounds__(256) col_stats_partial_kernel(const float* __restrict__ S,
                                                                float* __restrict__ part, int L,
                                                                int splits) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int split = blockIdx.y, b = blockIdx.z;
  if (j >= L) return;
  const int chunk = (L + splits - 1) / splits;
  const int i0 = split * chunk, i1 = min(L, i0 + chunk);
  const float* p = S + static_cast<size_t>(b) * L * L + j;
  float m = -INFINITY;
  for (int i = i0; i < i1; ++i) m = fmaxf(m, p[static_cast<size_t>(i) * L]);
  float s = 0.f;
  for (int i = i0; i < i1; ++i) s += __expf(__fsub_rn(p[static_cast<size_t>(i) * L], m));
  float* o = part + ((static_cast<size_t>(b) * splits + split) * L + j) * 2;
  o[0] = m;
  o[1] = s;
}
__global__ void col_stats_combine_kernel(const float* __restrict__ part, float* __restrict__ col_max,
                                         float* __restrict__ col_rsum, int L, int splits) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (j >= L) return;
  float m = -INFINITY;
  for (int k = 0; k < splits; ++k)
    m = fmaxf(m, part[((static_cast<size_t>(b) * splits + k) * L + j) * 2]);
  float s = 0.f;
  for (int k = 0; k < splits; ++k) {
    const float* q = part + ((static_cast<size_t>(b) * splits + k) * L + j) * 2;
    if (q[0] > -INFINITY) s += q[1] * __expf(q[0] - m);
  }
  col_max[static_cast<size_t>(b) * L + j] = m;
  col_rsum[static_cast<size_t>(b) * L + j] = 1.f / s;
}

__global__ void __launch_bounds__(256) row_conf_kernel(const float* __restrict__ S,
                                                       const float* __restrict__ row_max,
                                                       const float* __restrict__ row_rsum,
                                                       const float* __restrict__ col_max,
                                                       const float* __restrict__ col_rsum,
                                                       float* __restrict__ rconf_max,
                                                       int* __restrict__ rconf_arg,
                                                       int* __restrict__ rconf_ties, int L, bool raw) {
  __shared__ float sh[8];
  __shared__ int shi[8];
  const int b = blockIdx.y;
  const size_t r = static_cast<size_t>(b) * L + blockIdx.x;
  const float* p = S + r * L;
  const float rm = raw ? 0.f : row_max[r], rr = raw ? 0.f : row_rsum[r];
  const float* cm = col_max + static_cast<size_t>(b) * L;
  const float* cr = col_rsum + static_cast<size_t>(b) * L;
  float best = -1.f;
  int arg = 0x7fffffff;
  for (int j = threadIdx.x; j < L; j += 256) {
    const float c = conf_value(p[j], rm, rr, raw ? 0.f : cm[j], raw ? 0.f : cr[j], raw);
    if (c > best) { best = c; arg = j; }
  }
  const float bm = block_max_256(best, sh);
  // first index attaining the max, and how many attain it
  int cand = (best == bm) ? arg : 0x7fffffff;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
  if ((threadIdx.x & 31) == 0) shi[threadIdx.x >> 5] = cand;
  __syncthreads();
  int first = shi[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) first = min(first, shi[k]);
  __syncthreads();
  int ties = 0;
  for (int j = threadIdx.x; j < L; j += 256)
    ties += (conf_value(p[j], rm, rr, raw ? 0.f : cm[j], raw ? 0.f : cr[j], raw) == bm) ? 1 : 0;
  const float tsum = block_sum_256(static_cast<float>(ties), sh);
  if (threadIdx.x == 0) {
    rconf_max[r] = bm;
    rconf_arg[r] = first;
    rconf_ties[r] = static_cast<int>(tsum + 0.5f);
  }
}

__global__ void __launch_bounds__(256) col_conf_partial_kernel(const float* __restrict__ S,
                                                               const float* __restrict__ row_max,
                                                               const float* __restrict__ row_rsum,
                                                               const float* __restrict__ col_max,
                                                               const float* __restrict__ col_rsum,
                                                               float* __restrict__ part, int L,
                                                               int splits, bool raw) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  const int split = blockIdx.y, b = blockIdx.z;
  if (j >= L) return;
  const int chunk = (L + splits - 1) / splits;
  const int i0 = split * chunk, i1 = min(L, i0 + chunk);
  const float* p = S + static_cast<size_t>(b) * L * L + j;
  const float cm = raw ? 0.f : col_max[static_cast<size_t>(b) * L + j];
  const float cr = raw ? 0.f : col_rsum[static_cast<size_t>(b) * L + j];
  const float* rm = row_max + static_cast<size_t>(b) * L;
  const float* rr = row_rsum + static_cast<size_t>(b) * L;
  float best = -1.f;
  for (int i = i0; i < i1; ++i)
    best = fmaxf(best, conf_value(p[static_cast<size_t>(i) * L], raw ? 0.f : rm[i], raw ? 0.f : rr[i], cm, cr, raw));
  part[(static_cast<size_t>(b) * splits + split) * L + j] = best;
}
__global__ void col_conf_combine_kernel(const float* __restrict__ part, float* __restrict__ cconf_max,
                                        int L, int splits) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (j >= L) return;
  float m = -1.f;
  for (int k = 0; k < splits; ++k) m = fmaxf(m, part[(static_cast<size_t>(b) * splits + k) * L + j]);
  cconf_max[static_cast<size_t>(b) * L + j] = m;
}

// ---- fused passes (L % 4 == 0, L <= 6144): S is read from DRAM twice instead of four times.
// A block owns a slab of rows and all columns; thread t holds float4 column groups t, t+256, ... (6 per row).
//   stats_fused : row (max, 1/sum exp) per row + online per-column (max, sum exp) partials of the slab
//   conf_fused  : conf = softmax_row * softmax_col per element; row max / first argmax / tie count,
//                 per-column partial max of the slab
constexpr int kCmThreads = 512;   // 16 warps per block: the passes stream S with ~100 loads in flight per thread-pair
constexpr int kF4 = 3;            // float4 groups per thread per row (kCmThreads * 4 * kF4 >= L)

constexpr int kCmWarps = kCmThreads / 32;
template <int NV, bool IS_MAX>
__device__ __forceinline__ void block_reduce_n(float (&v)[NV], float* sh /* [NV][kCmWarps] */) {
#pragma unroll
  for (int q = 0; q < NV; ++q) v[q] = IS_MAX ? warp_max(v[q]) : warp_sum(v[q]);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) sh[q * kCmWarps + (threadIdx.x >> 5)] = v[q];
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < NV; ++q) {
    float r = sh[q * kCmWarps];
#pragma unroll
    for (int k = 1; k < kCmWarps; ++k) r = IS_MAX ? fmaxf(r, sh[q * kCmWarps + k]) : r + sh[q * kCmWarps + k];
    v[q] = r;
  }
  __syncthreads();
}

// The rows of S stream through a thread-private multi-stage cp.async ring in shared memory (every thread copies and
// later reads exactly its own 16-byte chunks, so no block barrier is involved): ~150 KB of loads stay in flight per SM
// while the previous rows are reduced, instead of a load phase and a compute phase taking turns.
constexpr int kCmStageBytes = 196608;   // stats: 2 stages x 4 rows, conf: 4 stages x 2 rows, of kF4 * kCmThreads float4
template <int R>
__device__ __forceinline__ void cm_issue(float4* stage, const float4* __restrict__ Sb, int i, int i1, int L4, int t) {
#pragma unroll
  for (int r = 0; r < R; ++r) {
#pragma unroll
    for (int k = 0; k < kF4; ++k) {
      const int f = t + kCmThreads * k;
      if (i + r < i1 && f < L4) cp_async16(stage + (r * kF4 + k) * kCmThreads + t, Sb + static_cast<size_t>(i + r) * L4 + f, true);
    }
  }
  cp_async_commit();
}

__global__ void __launch_bounds__(kCmThreads) stats_fused_kernel(const float* __restrict__ S, float* __restrict__ row_max,
                                                          float* __restrict__ row_rsum, float* __restrict__ part,
                                                          int L, int rows_per_block, int splits) {
  constexpr int R = 4;
  __shared__ float sh[R * kCmWarps];
  const int b = blockIdx.y, t = threadIdx.x;
  const int i0 = blockIdx.x * rows_per_block, i1 = min(L, i0 + rows_per_block);
  const int L4 = L >> 2;
  const float4* Sb = reinterpret_cast<const float4*>(S + static_cast<size_t>(b) * L * L);
  float cm[kF4 * 4], cs[kF4 * 4];
#pragma unroll
  for (int c = 0; c < kF4 * 4; ++c) { cm[c] = -INFINITY; cs[c] = 0.f; }
  const float4 ninf = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  extern __shared__ float4 cm_stage[];
  constexpr int STAGES = 2, kStageF4 = R * kF4 * kCmThreads;
  static_assert(STAGES * kStageF4 * 16 == kCmStageBytes, "ring size");
#pragma unroll
  for (int s_ = 0; s_ < STAGES - 1; ++s_) cm_issue<R>(cm_stage + s_ * kStageF4, Sb, i0 + s_ * R, i1, L4, t);
  int stg = 0;
  for (int i = i0; i < i1; i += R) {
    cm_issue<R>(cm_stage + ((stg + STAGES - 1) % STAGES) * kStageF4, Sb, i + (STAGES - 1) * R, i1, L4, t);
    cp_async_wait<STAGES - 1>();
    const float4* cur = cm_stage + stg * kStageF4;
    stg = (stg + 1) % STAGES;
    float4 v[R][kF4];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int k = 0; k < kF4; ++k) {
        const int f = t + kCmThreads * k;
        v[r][k] = (i + r < i1 && f < L4) ? cur[(r * kF4 + k) * kCmThreads + t] : ninf;
      }
    float rm[R], rs[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float m = -INFINITY;
#pragma unroll
      for (int k = 0; k < kF4; ++k) m = fmaxf(fmaxf(m, fmaxf(v[r][k].x, v[r][k].y)), fmaxf(v[r][k].z, v[r][k].w));
      rm[r] = m;
    }
    block_reduce_n<R, true>(rm, sh);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float a = 0.f;
      if (i + r < i1) {
#pragma unroll
        for (int k = 0; k < kF4; ++k) {
          a += __expf(__fsub_rn(v[r][k].x, rm[r])); a += __expf(__fsub_rn(v[r][k].y, rm[r]));
          a += __expf(__fsub_rn(v[r][k].z, rm[r])); a += __expf(__fsub_rn(v[r][k].w, rm[r]));
        }
      }
      rs[r] = a;
    }
    block_reduce_n<R, false>(rs, sh);
    if (t < R && i + t < i1) {
      row_max[static_cast<size_t>(b) * L + i + t] = rm[t];
      row_rsum[static_cast<size_t>(b) * L + i + t] = 1.f / rs[t];
    }
    // online per-column (max, sum exp) over these R rows
#pragma unroll
    for (int k = 0; k < kF4; ++k) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float x[R];
#pragma unroll
        for (int r = 0; r < R; ++r) x[r] = e == 0 ? v[r][k].x : e == 1 ? v[r][k].y : e == 2 ? v[r][k].z : v[r][k].w;
        float m4 = x[0];
#pragma unroll
        for (int r = 1; r < R; ++r) m4 = fmaxf(m4, x[r]);
        const int c = k * 4 + e;
        const float mn = fmaxf(cm[c], m4);
        if (mn > -INFINITY) {
          float a = cs[c] * __expf(cm[c] - mn);
#pragma unroll
          for (int r = 0; r < R; ++r) a += __expf(x[r] - mn);
          cs[c] = a;
          cm[c] = mn;
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kF4; ++k) {
    const int f = t + kCmThreads * k;
    if (f < L4) {
      float* o = part + ((static_cast<size_t>(b) * splits + blockIdx.x) * L + 4 * f) * 2;
#pragma unroll
      for (int e = 0; e < 4; ++e) { o[2 * e] = cm[k * 4 + e]; o[2 * e + 1] = cs[k * 4 + e]; }
    }
  }
}

__global__ void __launch_bounds__(kCmThreads) conf_fused_kernel(const float* __restrict__ S, const float* __restrict__ row_max,
                                                         const float* __restrict__ row_rsum,
                                                         const float* __restrict__ col_max,
                                                         const float* __restrict__ col_rsum,
                                                         float* __restrict__ rconf_max, int* __restrict__ rconf_arg,
                                                         int* __restrict__ rconf_ties, float* __restrict__ part,
                                                         int L, int rows_per_block, int splits, bool raw, float thr) {
  // Only entries with conf > thr can become matches (coarse_matching.py:183), and conf = p_row * p_col with both factors
  // <= 1, so conf > thr needs p_row > thr AND p_col > thr, i.e. S > max + ln(thr * sum) on the row and on the column side.
  // Everything else is skipped after two compares (at most 1 / thr entries of a row pass): the row / column maxima then run
  // over the candidates only, which changes them exactly where they are <= thr — where no match is possible anyway. With
  // thr <= 0 (or a raw confidence matrix) every entry is a candidate and the pass is the exhaustive one.
  constexpr int R = 2;
  constexpr float kSlack = 1e-3f;      // the screen is applied to S, the decision to the rounded conf: keep borderline entries
  const bool screen = thr > 0.f && !raw;
  __shared__ float sh[2 * R * kCmWarps];
  const int b = blockIdx.y, t = threadIdx.x;
  const int i0 = blockIdx.x * rows_per_block, i1 = min(L, i0 + rows_per_block);
  const int L4 = L >> 2;
  const float4* Sb = reinterpret_cast<const float4*>(S + static_cast<size_t>(b) * L * L);
  float4 cmv[kF4], crv[kF4], tcv[kF4];
  float cbest[kF4 * 4];
#pragma unroll
  for (int k = 0; k < kF4; ++k) {
    const int f = t + kCmThreads * k;
    const bool ok = f < L4 && !raw;
    cmv[k] = ok ? __ldg(reinterpret_cast<const float4*>(col_max + static_cast<size_t>(b) * L) + f) : make_float4(0, 0, 0, 0);
    crv[k] = ok ? __ldg(reinterpret_cast<const float4*>(col_rsum + static_cast<size_t>(b) * L) + f) : make_float4(0, 0, 0, 0);
    // column-side candidate bound: S > cmax + ln(thr / crs) - slack   (crs = 1 / sum)
    tcv[k] = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    if (screen && ok) {
      tcv[k].x = cmv[k].x + __logf(thr / crv[k].x) - kSlack; tcv[k].y = cmv[k].y + __logf(thr / crv[k].y) - kSlack;
      tcv[k].z = cmv[k].z + __logf(thr / crv[k].z) - kSlack; tcv[k].w = cmv[k].w + __logf(thr / crv[k].w) - kSlack;
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) cbest[k * 4 + e] = -1.f;
  }
  extern __shared__ float4 cm_stage[];
  constexpr int STAGES = 4, kStageF4 = R * kF4 * kCmThreads;
  static_assert(STAGES * kStageF4 * 16 == kCmStageBytes, "ring size");
#pragma unroll
  for (int s_ = 0; s_ < STAGES - 1; ++s_) cm_issue<R>(cm_stage + s_ * kStageF4, Sb, i0 + s_ * R, i1, L4, t);
  int stg = 0;
  for (int i = i0; i < i1; i += R) {
    cm_issue<R>(cm_stage + ((stg + STAGES - 1) % STAGES) * kStageF4, Sb, i + (STAGES - 1) * R, i1, L4, t);
    cp_async_wait<STAGES - 1>();
    const float4* cur = cm_stage + stg * kStageF4;
    stg = (stg + 1) % STAGES;
    float4 v[R][kF4];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int k = 0; k < kF4; ++k) {
        const int f = t + kCmThreads * k;
        v[r][k] = (i + r < i1 && f < L4) ? cur[(r * kF4 + k) * kCmThreads + t] : make_float4(0, 0, 0, 0);
      }
    float best[R];
    int arg[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const bool rok = i + r < i1;
      const size_t row = static_cast<size_t>(b) * L + (rok ? i + r : i);
      const float rmx = raw ? 0.f : row_max[row], rrs = raw ? 0.f : row_rsum[row];
      const float tr = screen ? rmx + __logf(thr / rrs) - kSlack : -INFINITY;      // row-side candidate bound
      best[r] = -1.f;
      arg[r] = 0x7fffffff;
#pragma unroll
      for (int k = 0; k < kF4; ++k) {
        const int f = t + kCmThreads * k;
        const bool ok = rok && f < L4;
        const float4 s4 = v[r][k];
        const bool c0 = ok && s4.x > tr && s4.x > tcv[k].x, c1 = ok && s4.y > tr && s4.y > tcv[k].y;
        const bool c2 = ok && s4.z > tr && s4.z > tcv[k].z, c3 = ok && s4.w > tr && s4.w > tcv[k].w;
        float4 c = make_float4(-1.f, -1.f, -1.f, -1.f);
        if (c0 | c1 | c2 | c3) {
          if (c0) c.x = conf_value(s4.x, rmx, rrs, cmv[k].x, crv[k].x, raw);
          if (c1) c.y = conf_value(s4.y, rmx, rrs, cmv[k].y, crv[k].y, raw);
          if (c2) c.z = conf_value(s4.z, rmx, rrs, cmv[k].z, crv[k].z, raw);
          if (c3) c.w = conf_value(s4.w, rmx, rrs, cmv[k].w, crv[k].w, raw);
          if (c.x > best[r]) { best[r] = c.x; arg[r] = 4 * f; }
          if (c.y > best[r]) { best[r] = c.y; arg[r] = 4 * f + 1; }
          if (c.z > best[r]) { best[r] = c.z; arg[r] = 4 * f + 2; }
          if (c.w > best[r]) { best[r] = c.w; arg[r] = 4 * f + 3; }
          cbest[k * 4] = fmaxf(cbest[k * 4], c.x); cbest[k * 4 + 1] = fmaxf(cbest[k * 4 + 1], c.y);
          cbest[k * 4 + 2] = fmaxf(cbest[k * 4 + 2], c.z); cbest[k * 4 + 3] = fmaxf(cbest[k * 4 + 3], c.w);
        }
        v[r][k] = c;   // keep the confidences for the tie count
      }
    }
    float bm[R];
#pragma unroll
    for (int r = 0; r < R; ++r) bm[r] = best[r];
    block_reduce_n<R, true>(bm, sh);
    // first index attaining the max (max of the negated candidate), and how many attain it
    float q[2 * R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      q[r] = (best[r] == bm[r] && arg[r] != 0x7fffffff) ? -static_cast<float>(arg[r]) : -INFINITY;   // indices < 2^24: exact
      int ties = 0;
      if (bm[r] >= 0.f) {               // a row without candidates has no maximum to tie with
#pragma unroll
        for (int k = 0; k < kF4; ++k)
          ties += (v[r][k].x == bm[r]) + (v[r][k].y == bm[r]) + (v[r][k].z == bm[r]) + (v[r][k].w == bm[r]);
      }
      q[R + r] = static_cast<float>(ties);
    }
    {  // one barrier pair for both reductions: max over q[0..R), sum over q[R..2R)
#pragma unroll
      for (int r = 0; r < R; ++r) { q[r] = warp_max(q[r]); q[R + r] = warp_sum(q[R + r]); }
      if ((t & 31) == 0) {
#pragma unroll
        for (int z = 0; z < 2 * R; ++z) sh[z * kCmWarps + (t >> 5)] = q[z];
      }
      __syncthreads();
      if (t < R && i + t < i1) {
        float fm = sh[t * kCmWarps], ts = sh[(R + t) * kCmWarps];
#pragma unroll
        for (int k = 1; k < kCmWarps; ++k) { fm = fmaxf(fm, sh[t * kCmWarps + k]); ts += sh[(R + t) * kCmWarps + k]; }
        const size_t row = static_cast<size_t>(b) * L + i + t;
        rconf_max[row] = bm[t];
        rconf_arg[row] = static_cast<int>(-fm);
        rconf_ties[row] = static_cast<int>(ts + 0.5f);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int k = 0; k < kF4; ++k) {
    const int f = t + kCmThreads * k;
    if (f < L4)
      *reinterpret_cast<float4*>(part + (static_cast<size_t>(b) * splits + blockIdx.x) * L + 4 * f) =
          make_float4(cbest[k * 4], cbest[k * 4 + 1], cbest[k * 4 + 2], cbest[k * 4 + 3]);
  }
}

__device__ __forceinline__ bool border_ok(int idx, int h, int w, int bd) {
  const int y = idx / w, x = idx - y * w;
  return y >= bd && y < h - bd && x >= bd && x < w - bd;
}

__global__ void select_kernel(const float* __restrict__ S, const float* __restrict__ row_max,
                              const float* __restrict__ row_rsum, const float* __restrict__ col_max,
                              const float* __restrict__ col_rsum, const float* __restrict__ rconf_max,
                              const int* __restrict__ rconf_arg, const int* __restrict__ rconf_ties,
                              const float* __restrict__ cconf_max, int* __restrict__ jsel, int L,
                              int h_c, int w_c, float thr, int border, bool raw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= L) return;
  const size_t r = static_cast<size_t>(b) * L + i;
  const float v = rconf_max[r];
  int sel = -1;
  if (v > thr && border_ok(i, h_c, w_c, border)) {
    const float* cc = cconf_max + static_cast<size_t>(b) * L;
    const int j = rconf_arg[r];
    if (border_ok(j, h_c, w_c, border) && v == cc[j]) {
      sel = j;
    } else if (rconf_ties[r] > 1) {
      // rare: several columns attain the row maximum; take the first that is also a column maximum
      const float* p = S + r * L;
      const float rm = raw ? 0.f : row_max[r], rr = raw ? 0.f : row_rsum[r];
      const float* cm = col_max + static_cast<size_t>(b) * L;
      const float* cr = col_rsum + static_cast<size_t>(b) * L;
      for (int jj = j + 1; jj < L; ++jj) {
        const float c = conf_value(p[jj], rm, rr, raw ? 0.f : cm[jj], raw ? 0.f : cr[jj], raw);
        if (c == v && c == cc[jj] && border_ok(jj, h_c, w_c, border)) { sel = jj; break; }
      }
    }
  }
  jsel[r] = sel;
}

// single block: ordered compaction over (b, i)
__global__ void __launch_bounds__(1024) compact_kernel(const int* __restrict__ jsel,
                                                       const float* __restrict__ rconf_max, int B, int L,
                                                       int w_c, float scale, int* __restrict__ m_total,
                                                       int* __restrict__ m_offsets, int* __restrict__ b_ids,
                                                       int* __restrict__ i_ids, int* __restrict__ j_ids,
                                                       float* __restrict__ mconf, float* __restrict__ mk0,
                                                       float* __restrict__ mk1) {
  __shared__ int wsum[32];
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int b = 0; b < B; ++b) {
    if (threadIdx.x == 0) m_offsets[b] = base;
    for (int i0 = 0; i0 < L; i0 += 1024) {
      const int i = i0 + threadIdx.x;
      int j = -1;
      if (i < L) j = jsel[static_cast<size_t>(b) * L + i];
      const int flag = j >= 0 ? 1 : 0;
      int inc = flag;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
      }
      if (lane == 31) wsum[wid] = inc;
      __syncthreads();
      if (wid == 0) {
        int w = wsum[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int t = __shfl_up_sync(0xffffffffu, w, o);
          if (lane >= o) w += t;
        }
        wsum[lane] = w;
      }
      __syncthreads();
      const int prefix = base + (wid > 0 ? wsum[wid - 1] : 0) + inc - flag;
      if (flag) {
        b_ids[prefix] = b;
        i_ids[prefix] = i;
        j_ids[prefix] = j;
        mconf[prefix] = rconf_max[static_cast<size_t>(b) * L + i];
        mk0[2 * prefix] = static_cast<float>(i % w_c) * scale;
        mk0[2 * prefix + 1] = static_cast<float>(i / w_c) * scale;
        mk1[2 * prefix] = static_cast<float>(j % w_c) * scale;
        mk1[2 * prefix + 1] = static_cast<float>(j / w_c) * scale;
      }
      __syncthreads();
      if (threadIdx.x == 0) base += wsum[31];
      __syncthreads();
    }
  }
  if (threadIdx.x == 0) {
    m_offsets[B] = base;
    m_total[0] = base;
    m_total[1] = 2 * base;
    m_total[2] = 25 * base;
    m_total[3] = 50 * base;
  }
}

// ------------------------------------------------------------------------------------------ fine level
__global__ void __launch_bounds__(64) fine_gather_coarse_kernel(const float* __restrict__ tok,
                                                                long long ldt, int B, int L,
                                                                const int* __restrict__ b_ids,
                                                                const int* __restrict__ i_ids,
                                                                const int* __restrict__ j_ids,
                                                                const int* __restrict__ m_total,
                                                                int Mcap, float* __restrict__ cin) {
  const int m = blockIdx.x, s = blockIdx.y;
  if (m >= m_total[0]) return;
  const int b = b_ids[m];
  const int tokidx = s == 0 ? i_ids[m] : j_ids[m];
  const size_t row = (static_cast<size_t>(s == 0 ? b : B + b)) * L + tokidx;
  const float4 v = *reinterpret_cast<const float4*>(tok + row * ldt + threadIdx.x * 4);
  *reinterpret_cast<float4*>(cin + (static_cast<size_t>(s) * Mcap + m) * 256 + threadIdx.x * 4) = v;
}

// dst[k][0:n16) = src[0:n16) for k = blockIdx.y (16-byte elements; grid-stride over x)
__global__ void __launch_bounds__(256) broadcast_copies_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                                               long long n16) {
  uint4* d = dst + static_cast<size_t>(blockIdx.y) * n16;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n16;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    d[i] = src[i];
}

__global__ void __launch_bounds__(128) fine_gather_windows_kernel(
    const float* __restrict__ featf0, long long img_stride0, const float* __restrict__ featf1, long long img_stride1,
    int Hf, int Wf, int w_c, int stride,
    const int* __restrict__ b_ids, const int* __restrict__ i_ids, const int* __restrict__ j_ids,
    const int* __restrict__ m_total, int Mcap, const float* __restrict__ cproj, float* __restrict__ win) {
  const int m = blockIdx.x, s = blockIdx.y;
  if (m >= m_total[0]) return;
  const int b = b_ids[m];
  const int idx = s == 0 ? i_ids[m] : j_ids[m];
  const int cy = idx / w_c, cx = idx - cy * w_c;
  const float* featf = s == 0 ? featf0 + b * img_stride0 : featf1 + b * img_stride1;
  const int c = threadIdx.x;
  const float cp = cproj[(static_cast<size_t>(s) * Mcap + m) * 128 + c];
  float* o = win + (static_cast<size_t>(s) * Mcap + m) * 25 * 256;
#pragma unroll 5
  for (int tap = 0; tap < 25; ++tap) {
    const int y = cy * stride - 2 + tap / 5, x = cx * stride - 2 + tap % 5;
    float v = 0.f;
    if (y >= 0 && y < Hf && x >= 0 && x < Wf)
      v = featf[(static_cast<size_t>(y) * Wf + x) * 128 + c];
    o[tap * 256 + c] = v;
    o[tap * 256 + 128 + c] = cp;
  }
}

__global__ void __launch_bounds__(128) fine_match_kernel(const float* __restrict__ f0,
                                                         const float* __restrict__ f1, long long ldf,
                                                         const float* __restrict__ mk1c,
                                                         const int* __restrict__ m_total, float scale_f,
                                                         float* __restrict__ mk1f, float* __restrict__ expec) {
  const int m = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (m >= m_total[0]) return;
  const int lane = threadIdx.x & 31;
  const float* c0 = f0 + (static_cast<size_t>(m) * 25 + 12) * ldf;
  float sim = -INFINITY;
  if (lane < 25) {
    const float* r1 = f1 + (static_cast<size_t>(m) * 25 + lane) * ldf;
    float a = 0.f;
#pragma unroll 8
    for (int k = 0; k < 32; ++k) {
      const float4 u = *reinterpret_cast<const float4*>(c0 + 4 * k);
      const float4 w = *reinterpret_cast<const float4*>(r1 + 4 * k);
      a = fmaf(u.x, w.x, a); a = fmaf(u.y, w.y, a); a = fmaf(u.z, w.z, a); a = fmaf(u.w, w.w, a);
    }
    sim = a * 0.08838834764831845f;  // 1/sqrt(128)
  }
  const float mx = warp_max(sim);
  const float e = lane < 25 ? __expf(sim - mx) : 0.f;
  const float heat = e / warp_sum(e);
  const float gx = -1.f + 0.5f * (lane % 5), gy = -1.f + 0.5f * (lane / 5);
  const float ex = warp_sum(heat * gx), ey = warp_sum(heat * gy);
  const float vx = warp_sum(heat * gx * gx) - ex * ex, vy = warp_sum(heat * gy * gy) - ey * ey;
  if (lane == 0) {
    mk1f[2 * m] = mk1c[2 * m] + ex * 2.f * scale_f;
    mk1f[2 * m + 1] = mk1c[2 * m + 1] + ey * 2.f * scale_f;
    expec[3 * m] = ex;
    expec[3 * m + 1] = ey;
    expec[3 * m + 2] = sqrtf(fmaxf(vx, 1e-10f)) + sqrtf(fmaxf(vy, 1e-10f));
  }
}


// ------------------------------------------------------------------------------------------ stem on mma.sync (bf16 x 3)
// The 7x7 stride-2 stem (1 -> 128 channels, resnet_fpn.py:52-54) as an implicit GEMM on warp-level tensor cores:
// M = 16 output pixels of one row, N = 32 channels per warp, K = 8 ky x 8 kx (row ky = 7 and tap kx = 7 carry zero
// weights, so two consecutive K elements are two consecutive image pixels and every A register is one aligned 32-bit
// shared-memory load). fp32 accuracy is kept by splitting image and weights into bf16 hi + lo parts and accumulating
// hi*hi + hi*lo + lo*hi in fp32 (error ~2^-16 relative, below TF32). Block = one output row of one image.
constexpr bool kUseMmaStem = true;
template <bool OBF>
__global__ void __launch_bounds__(128) stem_mma_kernel(const float* __restrict__ img, const float* __restrict__ w,
                                                       const float* __restrict__ bias, void* __restrict__ out,
                                                       int H, int W, int Ho, int Wo, int PW) {
  extern __shared__ __align__(16) unsigned short stem_sm[];       // [2 (hi, lo)][8 rows][PW]
  const int n = blockIdx.y, y = blockIdx.x;
  const int t = threadIdx.x, wid = t >> 5, lane = t & 31, g = lane >> 2, tq = lane & 3;
  unsigned short* p_hi = stem_sm;
  unsigned short* p_lo = stem_sm + 8 * PW;
  for (int idx = t; idx < 8 * PW; idx += 128) {
    const int ky = idx / PW, col = idx - ky * PW;
    const int iy = 2 * y - 3 + ky, ix = col - 3;
    float v = 0.f;
    if (ky < 7 && iy >= 0 && iy < H && ix >= 0 && ix < W) v = img[(static_cast<size_t>(n) * H + iy) * W + ix];
    const unsigned short hi = f2bf(v);
    p_hi[idx] = hi;
    p_lo[idx] = f2bf(v - bf2f(hi));
  }
  // B fragments of this warp's 32 channels: k = 16 ks + {2 tq, 2 tq + 1} -> (ky = 2 ks, kx = 2 tq + {0, 1}); + 8 -> ky = 2 ks + 1
  unsigned bh[4][4][2], bl[4][4][2];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    const float* wc = w + (32 * wid + 8 * nt + g) * 49;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int ky = 2 * ks + half, kx = 2 * tq;
        const float w0 = ky < 7 ? wc[ky * 7 + kx] : 0.f;
        const float w1 = (ky < 7 && kx + 1 < 7) ? wc[ky * 7 + kx + 1] : 0.f;
        const unsigned short h0 = f2bf(w0), h1 = f2bf(w1);
        bh[nt][ks][half] = static_cast<unsigned>(h0) | (static_cast<unsigned>(h1) << 16);
        bl[nt][ks][half] = pack_bf16(w0 - bf2f(h0), w1 - bf2f(h1));
      }
    }
  }
  float bia[4][2];
#pragma unroll
  for (int nt = 0; nt < 4; ++nt) {
    bia[nt][0] = bias[32 * wid + 8 * nt + 2 * tq];
    bia[nt][1] = bias[32 * wid + 8 * nt + 2 * tq + 1];
  }
  __syncthreads();
  const int mtiles = (Wo + 15) / 16;
  for (int mt = 0; mt < mtiles; ++mt) {
    float acc[4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
    }
    const int c_lo = 2 * (16 * mt + g) + 2 * tq;        // patch column of (pixel row g, kx = 2 tq)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      unsigned ah[4], al[4];
      const int r0 = (2 * ks) * PW, r1 = (2 * ks + 1) * PW;
      ah[0] = *reinterpret_cast<const unsigned*>(p_hi + r0 + c_lo);
      ah[1] = *reinterpret_cast<const unsigned*>(p_hi + r0 + c_lo + 16);
      ah[2] = *reinterpret_cast<const unsigned*>(p_hi + r1 + c_lo);
      ah[3] = *reinterpret_cast<const unsigned*>(p_hi + r1 + c_lo + 16);
      al[0] = *reinterpret_cast<const unsigned*>(p_lo + r0 + c_lo);
      al[1] = *reinterpret_cast<const unsigned*>(p_lo + r0 + c_lo + 16);
      al[2] = *reinterpret_cast<const unsigned*>(p_lo + r1 + c_lo);
      al[3] = *reinterpret_cast<const unsigned*>(p_lo + r1 + c_lo + 16);
#pragma unroll
      for (int nt = 0; nt < 4; ++nt) {
        mma_bf16(acc[nt], al, bh[nt][ks][0], bh[nt][ks][1]);
        mma_bf16(acc[nt], ah, bl[nt][ks][0], bl[nt][ks][1]);
        mma_bf16(acc[nt], ah, bh[nt][ks][0], bh[nt][ks][1]);
      }
    }
    const int x_lo = 16 * mt + g;
    const size_t row = (static_cast<size_t>(n) * Ho + y) * Wo;
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
      const int c = 32 * wid + 8 * nt + 2 * tq;
      const float o0 = fmaxf(acc[nt][0] + bia[nt][0], 0.f), o1 = fmaxf(acc[nt][1] + bia[nt][1], 0.f);
      const float o2 = fmaxf(acc[nt][2] + bia[nt][0], 0.f), o3 = fmaxf(acc[nt][3] + bia[nt][1], 0.f);
      if constexpr (OBF) {
        unsigned short* o = static_cast<unsigned short*>(out);
        if (x_lo < Wo) *reinterpret_cast<unsigned*>(o + (row + x_lo) * 128 + c) = pack_bf16(o0, o1);
        if (x_lo + 8 < Wo) *reinterpret_cast<unsigned*>(o + (row + x_lo + 8) * 128 + c) = pack_bf16(o2, o3);
      } else {
        float* o = static_cast<float*>(out);
        if (x_lo < Wo) *reinterpret_cast<float2*>(o + (row + x_lo) * 128 + c) = make_float2(o0, o1);
        if (x_lo + 8 < Wo) *reinterpret_cast<float2*>(o + (row + x_lo + 8) * 128 + c) = make_float2(o2, o3);
      }
    }
  }
}

}  // namespace

// ================================================================================================
// launch wrappers
// ================================================================================================
int stem_conv7x7(const float* img, const float* w, const float* bias, float* out, int NI, int H, int W,
                 cudaStream_t st, int out_bf16, int exact_fp32) {
  const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
  if (kUseMmaStem && !exact_fp32) {
    const int PW = 32 * ((Wo + 15) / 16) + 8;                 // patch columns: 2 px + kx for every pixel of the padded row
    const int smem = 2 * 8 * PW * 2;
    if (smem <= 48 * 1024) {
      if (out_bf16) stem_mma_kernel<true><<<dim3(Ho, NI), 128, smem, st>>>(img, w, bias, out, H, W, Ho, Wo, PW);
      else stem_mma_kernel<false><<<dim3(Ho, NI), 128, smem, st>>>(img, w, bias, out, H, W, Ho, Wo, PW);
      MFR_CUDA_CHECK(cudaGetLastError());
      return MFR_OK;
    }
  }
  dim3 grid((Wo + kStemPx - 1) / kStemPx, Ho, NI);
  if (out_bf16) stem_kernel<true><<<grid, 128, 0, st>>>(img, w, bias, out, H, W, Ho, Wo);
  else stem_kernel<false><<<grid, 128, 0, st>>>(img, w, bias, out, H, W, Ho, Wo);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int upsample2x_add(const void* src, void* dst, int N, int Hs, int Ws, int C, int lds, int ldd, int src_bf16,
                   int dst_bf16, cudaStream_t st) {
  if (C % 4 || lds % 4 || ldd % 4) return MFR_ERR_ARG;
  const int Hd = 2 * Hs, Wd = 2 * Ws;
  const float ry = Hd > 1 ? static_cast<float>(Hs - 1) / static_cast<float>(Hd - 1) : 0.f;
  const float rx = Wd > 1 ? static_cast<float>(Ws - 1) / static_cast<float>(Wd - 1) : 0.f;
  const size_t total = static_cast<size_t>(N) * Hd * Wd * (C / 4);
  const unsigned g = static_cast<unsigned>((total + 255) / 256);
  if (dst_bf16 && (ldd % 8 == 0) && (lds % (src_bf16 ? 8 : 4) == 0) && (C + 7) / 8 * 8 <= ldd && (C + 7) / 8 * 8 <= lds) {
    const int C8 = (C + 7) / 8;
    const dim3 g8(static_cast<unsigned>((Wd * C8 + 255) / 256), static_cast<unsigned>(Hd), static_cast<unsigned>(N));
    if (src_bf16) upsample2x_add8_kernel<true><<<g8, 256, 0, st>>>(src, dst, Hs, Ws, C8, lds, ldd, ry, rx);
    else upsample2x_add8_kernel<false><<<g8, 256, 0, st>>>(src, dst, Hs, Ws, C8, lds, ldd, ry, rx);
  } else if (src_bf16 && dst_bf16) upsample2x_add_kernel<true, true><<<g, 256, 0, st>>>(src, dst, N, Hs, Ws, C / 4, lds, ldd, ry, rx);
  else if (!src_bf16 && dst_bf16) upsample2x_add_kernel<false, true><<<g, 256, 0, st>>>(src, dst, N, Hs, Ws, C / 4, lds, ldd, ry, rx);
  else if (!src_bf16 && !dst_bf16) upsample2x_add_kernel<false, false><<<g, 256, 0, st>>>(src, dst, N, Hs, Ws, C / 4, lds, ldd, ry, rx);
  else return MFR_ERR_UNSUPPORTED;
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int weights_to_bf16(const float* src, void* dst, size_t rows, int cin, int cin_pad, cudaStream_t st) {
  const size_t total = rows * cin_pad;
  weights_to_bf16_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
      src, static_cast<unsigned short*>(dst), rows, cin, cin_pad);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int posenc_tokens(const float* feat, const float* pe, float* tok, long long ldt, int N, int L, int C,
                  cudaStream_t st) {
  const size_t total = static_cast<size_t>(N) * L * (C / 4);
  posenc_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(feat, pe, tok, ldt, N, L,
                                                                           C / 4);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int linear_attention_long(const void* Q, long long ldq, const void* K, long long ldk, const void* V,
                          long long ldv, void* msg, long long ldm, float* kv_part, float* kv, int n,
                          int L, int S, int heads, int dim, int splits, cudaStream_t st, int bf16) {
  if (dim != 32 || heads != 8) return MFR_ERR_UNSUPPORTED;
  if ((ldq | ldk | ldv) & (bf16 ? 7 : 3)) return MFR_ERR_ARG;                    // 16-byte cp.async chunks
  constexpr int kKvSmem = 2 * kAttStages * kSlab * 256 * 4, kApSmem = kAttStages * kSlab * 256 * 4;
  static bool attr_seen[64] = {};
  if (first_call_on_device(attr_seen)) {
    MFR_CUDA_CHECK(cudaFuncSetAttribute(kv_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kKvSmem));
    MFR_CUDA_CHECK(cudaFuncSetAttribute(attn_apply_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kApSmem));
    MFR_CUDA_CHECK(cudaFuncSetAttribute(kv_partial_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * kMStages * kMSlabBytes));
    MFR_CUDA_CHECK(cudaFuncSetAttribute(attn_apply_mma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMStages * kMSlabBytes));
  }
  if (bf16) {
    const int msplits = std::max(1, std::min((L + kMS - 1) / kMS, (4 * sm_count() + n - 1) / n));
    kv_partial_mma_kernel<<<dim3(splits, n), 256, 2 * kMStages * kMSlabBytes, st>>>(K, ldk, V, ldv, kv_part, S, splits);
    kv_reduce_kernel<<<dim3((8 * 1056 + 255) / 256, n), 256, 0, st>>>(kv_part, kv, splits);
    attn_apply_mma_kernel<<<dim3(msplits, n), 256, kMStages * kMSlabBytes, st>>>(Q, ldq, kv, static_cast<unsigned short*>(msg), ldm, L,
                                                                               1e-6f, msplits);
  } else {
    const int asplits = std::max(1, std::min((L + kSlab - 1) / kSlab, (4 * sm_count() + n - 1) / n));
    kv_partial_kernel<<<dim3(splits, n), 256, kKvSmem, st>>>(K, ldk, V, ldv, kv_part, S, splits);
    kv_reduce_kernel<<<dim3((8 * 1056 + 255) / 256, n), 256, 0, st>>>(kv_part, kv, splits);
    attn_apply_kernel<<<dim3(asplits, n), 256, kApSmem, st>>>(Q, ldq, kv, msg, ldm, L, S, 1e-6f, asplits);
  }
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int linear_attention_windows(const void* Q, long long ldq, const void* K, long long ldk, const void* V,
                             long long ldv, void* msg, long long ldm, const int* n_items_dev,
                             int max_items, int T, cudaStream_t st, int bf16) {
  if (T != 25 || max_items <= 0) return MFR_ERR_UNSUPPORTED;
  if (bf16) {
    if ((ldq | ldk | ldv) & 7) return MFR_ERR_ARG;
    attn_windows_mma_kernel<25><<<max_items, 256, 0, st>>>(static_cast<const unsigned short*>(Q), ldq, static_cast<const unsigned short*>(K), ldk,
                                                           static_cast<const unsigned short*>(V), ldv, static_cast<unsigned short*>(msg), ldm,
                                                           n_items_dev, 1e-6f);
  } else {
    attn_windows_kernel<25><<<max_items, 128, 0, st>>>(Q, ldq, K, ldk, V, ldv, msg, ldm, n_items_dev, 1e-6f);
  }
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int layernorm_rows(const float* in, long long ldi, const float* gamma, const float* beta,
                   const float* res, long long ldr, float* out, long long ldo, long long rows, int C,
                   const int* dyn_rows, cudaStream_t st) {
  unsigned grid = static_cast<unsigned>(std::min<long long>((rows + 7) / 8, static_cast<long long>(sm_count()) * 16));
  if (grid == 0) return MFR_OK;
  if (out == nullptr) return MFR_ERR_ARG;
  if (C == 256)
    layernorm_kernel<256><<<grid, 256, 0, st>>>(in, ldi, gamma, beta, res, ldr, out, ldo, rows, dyn_rows);
  else if (C == 128)
    layernorm_kernel<128><<<grid, 256, 0, st>>>(in, ldi, gamma, beta, res, ldr, out, ldo, rows, dyn_rows);
  else
    return MFR_ERR_UNSUPPORTED;
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int rows_to_bf16(const float* src, long long lds, void* dst, long long ldd, long long rows, int C, const int* dyn_rows,
                 cudaStream_t st) {
  if ((C & 3) || (lds & 3) || (ldd & 3) || rows <= 0) return MFR_ERR_ARG;
  const long long total = rows * (C / 4);
  const unsigned grid = static_cast<unsigned>(std::min<long long>((total + 255) / 256, static_cast<long long>(sm_count()) * 16));
  rows_to_bf16_kernel<<<grid, 256, 0, st>>>(src, lds, static_cast<unsigned short*>(dst), ldd, rows, C / 4, dyn_rows);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int broadcast_copies(const void* src, long long bytes, void* dst, int copies, cudaStream_t st) {
  if ((bytes & 15) || (reinterpret_cast<uintptr_t>(src) & 15) || (reinterpret_cast<uintptr_t>(dst) & 15) || copies < 1)
    return MFR_ERR_ARG;
  const long long n16 = bytes / 16;
  const unsigned gx = static_cast<unsigned>(std::min<long long>((n16 + 255) / 256, std::max(1LL, static_cast<long long>(sm_count()) * 16 / copies)));
  broadcast_copies_kernel<<<dim3(gx, static_cast<unsigned>(copies)), 256, 0, st>>>(static_cast<const uint4*>(src),
                                                                                  static_cast<uint4*>(dst), n16);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int rows_split3(const float* src, long long lds, long long src_img_stride, float* dst, long long rows_per_img,
                int images, int C, int pattern, const int* dyn_rows, cudaStream_t st) {
  if ((C & 3) || (lds & 3) || (src_img_stride & 3) || rows_per_img <= 0 || images <= 0 || images > 65535) return MFR_ERR_ARG;
  const long long total = rows_per_img * (C / 4);
  const unsigned gx = static_cast<unsigned>(std::min<long long>((total + 255) / 256, std::max(1LL, static_cast<long long>(sm_count()) * 16 / images)));
  rows_split3_kernel<<<dim3(gx, static_cast<unsigned>(images)), 256, 0, st>>>(src, lds, src_img_stride, dst, rows_per_img,
                                                                             C / 4, pattern, dyn_rows);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int coarse_match(const float* S, CoarseMatchBuffers f, int B, int L, int h_c, int w_c, float thr,
                 int border, float scale, int splits, cudaStream_t st, bool input_is_conf) {
  const int cb = (L + 255) / 256;
  const bool raw = input_is_conf;
  const bool fused = (L % 4 == 0) && L <= kCmThreads * 4 * kF4 && (reinterpret_cast<uintptr_t>(S) & 15) == 0;
  if (fused) {
    static bool attr_seen[64] = {};
    if (first_call_on_device(attr_seen)) {
      MFR_CUDA_CHECK(cudaFuncSetAttribute(stats_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kCmStageBytes));
      MFR_CUDA_CHECK(cudaFuncSetAttribute(conf_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kCmStageBytes));
    }
    // a block owns ceil(L / splits) rows (rounded to the row batch) and all columns
    const int rpb = ((L + splits - 1) / splits + 3) / 4 * 4;
    const int nblk = (L + rpb - 1) / rpb;
    if (!raw) {
      stats_fused_kernel<<<dim3(nblk, B), kCmThreads, kCmStageBytes, st>>>(S, f.row_max, f.row_rsum, f.col_part, L, rpb, nblk);
      col_stats_combine_kernel<<<dim3(cb, B), 256, 0, st>>>(f.col_part, f.col_max, f.col_rsum, L, nblk);
    }
    conf_fused_kernel<<<dim3(nblk, B), kCmThreads, kCmStageBytes, st>>>(S, f.row_max, f.row_rsum, f.col_max, f.col_rsum, f.rconf_max,
                                                     f.rconf_arg, f.rconf_ties, f.col_part, L, rpb, nblk, raw, thr);
    col_conf_combine_kernel<<<dim3(cb, B), 256, 0, st>>>(f.col_part, f.cconf_max, L, nblk);
  } else {
    if (!raw) {
      row_stats_kernel<<<dim3(L, B), 256, 0, st>>>(S, f.row_max, f.row_rsum, L);
      col_stats_partial_kernel<<<dim3(cb, splits, B), 256, 0, st>>>(S, f.col_part, L, splits);
      col_stats_combine_kernel<<<dim3(cb, B), 256, 0, st>>>(f.col_part, f.col_max, f.col_rsum, L, splits);
    }
    row_conf_kernel<<<dim3(L, B), 256, 0, st>>>(S, f.row_max, f.row_rsum, f.col_max, f.col_rsum,
                                                f.rconf_max, f.rconf_arg, f.rconf_ties, L, raw);
    col_conf_partial_kernel<<<dim3(cb, splits, B), 256, 0, st>>>(S, f.row_max, f.row_rsum, f.col_max,
                                                                 f.col_rsum, f.col_part, L, splits, raw);
    col_conf_combine_kernel<<<dim3(cb, B), 256, 0, st>>>(f.col_part, f.cconf_max, L, splits);
  }
  select_kernel<<<dim3(cb, B), 256, 0, st>>>(S, f.row_max, f.row_rsum, f.col_max, f.col_rsum,
                                             f.rconf_max, f.rconf_arg, f.rconf_ties, f.cconf_max, f.jsel,
                                             L, h_c, w_c, thr, border, raw);
  compact_kernel<<<1, 1024, 0, st>>>(f.jsel, f.rconf_max, B, L, w_c, scale, f.m_total, f.m_offsets,
                                     f.b_ids, f.i_ids, f.j_ids, f.mconf, f.mkpts0_c, f.mkpts1_c);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

// row slabs per pair: the fused kernels run one block per SM (their cp.async ring fills the shared memory), so B * splits
// is kept at or just under two full waves of the SMs (rounding up would add a nearly empty third wave)
int coarse_match_splits(int B, int L) { return std::max(1, std::min((L + 3) / 4, (2 * sm_count()) / B)); }

int coarse_match_alloc(int B, int L, int splits, CoarseMatchBuffers* o) {
  const size_t BL = static_cast<size_t>(B) * L;
  memset(o, 0, sizeof(*o));
  bool ok = true;
  auto A = [&](void** p, size_t bytes) { ok &= cudaMalloc(p, bytes) == cudaSuccess; };
  A((void**)&o->row_max, BL * 4); A((void**)&o->row_rsum, BL * 4); A((void**)&o->col_max, BL * 4);
  A((void**)&o->col_rsum, BL * 4); A((void**)&o->col_part, BL * splits * 2 * 4);
  A((void**)&o->rconf_max, BL * 4); A((void**)&o->rconf_arg, BL * 4); A((void**)&o->rconf_ties, BL * 4);
  A((void**)&o->cconf_max, BL * 4); A((void**)&o->jsel, BL * 4); A((void**)&o->m_total, 16);
  A((void**)&o->m_offsets, (B + 1) * 4); A((void**)&o->b_ids, BL * 4); A((void**)&o->i_ids, BL * 4);
  A((void**)&o->j_ids, BL * 4); A((void**)&o->mconf, BL * 4); A((void**)&o->mkpts0_c, BL * 8);
  A((void**)&o->mkpts1_c, BL * 8);
  if (!ok) { coarse_match_free(o); return MFR_ERR_CUDA; }
  return MFR_OK;
}
void coarse_match_free(CoarseMatchBuffers* o) {
  void* ps[] = {o->row_max, o->row_rsum, o->col_max, o->col_rsum, o->col_part, o->rconf_max, o->rconf_arg,
                o->rconf_ties, o->cconf_max, o->jsel, o->m_total, o->m_offsets, o->b_ids, o->i_ids, o->j_ids,
                o->mconf, o->mkpts0_c, o->mkpts1_c};
  for (void* p : ps) if (p) cudaFree(p);
  memset(o, 0, sizeof(*o));
}

int fine_gather_coarse(const float* tok, long long ldt, int B, int L, const int* b_ids, const int* i_ids,
                       const int* j_ids, const int* m_total, int Mcap, float* cin, cudaStream_t st) {
  fine_gather_coarse_kernel<<<dim3(Mcap, 2), 64, 0, st>>>(tok, ldt, B, L, b_ids, i_ids, j_ids, m_total,
                                                          Mcap, cin);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int fine_gather_windows(const float* featf0, long long img_stride0, const float* featf1, long long img_stride1, int Hf,
                        int Wf, int w_c, const int* b_ids, const int* i_ids, const int* j_ids, const int* m_total,
                        int Mcap, const float* cproj, float* win, cudaStream_t st) {
  const int stride = Wf / w_c;
  fine_gather_windows_kernel<<<dim3(Mcap, 2), 128, 0, st>>>(featf0, img_stride0, featf1, img_stride1, Hf, Wf, w_c, stride,
                                                            b_ids, i_ids, j_ids, m_total, Mcap, cproj, win);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int fine_match(const float* f0, const float* f1, long long ldf, const float* mkpts1_c,
               const int* m_total, int Mcap, float scale_f, float* mkpts1_f, float* expec,
               cudaStream_t st) {
  fine_match_kernel<<<(Mcap + 3) / 4, 128, 0, st>>>(f0, f1, ldf, mkpts1_c, m_total, scale_f, mkpts1_f,
                                                    expec);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

}  // namespace mfr
