// csc.cu — fused BGRA / RGBA / BGR / RGB -> BT.709 limited-range NV12 colour conversion (+ bilinear scale), sm_90a.
//
// Replaces the colour-conversion stage of the reference's native capture module
// (pixelflux, call site src/selkies/media_pipeline.py:299-300; legacy GStreamer
// `videoconvert`, docs/component.md:338-344).  Integer spec: DESIGN.md §3; the CPU
// restatement it must match bit-for-bit is oracle/csc_ref.c.
//
// Roofline: HBM-bound streaming kernel, 4 B/px read + 1.5 B/px written (5.5 B/px algorithmic).
//   fast path  (1:1, width % 4 == 0): one thread = 4 px x 2 rows per unit: two 16-byte loads
//              (ld.global.nc.L1::no_allocate.v4), two 4-byte Y stores and one 4-byte CbCr store, all
//              warp-contiguous (512 B / 128 B / 128 B per warp instruction).  Two units per thread are
//              issued back to back so four 16-byte loads are in flight per thread.
//   arithmetic: dp2a (two 16-bit coefficient x 8-bit pixel MACs per instruction); rounding
//              constant and the +16 / +128 offsets are folded into the accumulator seed.
//   packed 3-byte path (BGR / RGB, 1:1, width % 16 == 0): one thread = 16 px x 2 rows: 4.5 B/px algorithmic.  A warp reads
//              its 1536 B of a row as three warp-contiguous 16-byte loads, trades them through shared memory so that each
//              thread holds its own 48 B, expands them to pixel words with byte permutes and stores 16 B of Y per row and
//              16 B of CbCr.
//   channel order: RGBA and RGB swap the coefficients of bytes 0 and 2 (at compile time in the 1:1 kernels, by matrix row in
//              the others); the pixels are never reordered.
//   planar 1:1 path (b2v_submit_tensor: three planes of uint8, fp16, bf16 or fp32 with contiguous rows): one thread = the
//              pixels of one 16-byte load (16 / 8 / 8 / 4) x 2 rows: six 16-byte loads, one per plane and row, all issued before
//              the first use; the elements are quantised in registers (DESIGN.md §3) and woven into the pixel words of the
//              4-byte kernel.  4.5 / 7.5 / 7.5 / 13.5 B/px algorithmic.  Which plane is blue is decided on the host.
//   general path (scaled or ragged widths): one thread per 2x2 output block, taps from tables.
//   any other tensor (interleaved floats, strided columns, unaligned windows, scaled): the general and scaled kernels, whose
//              per-pixel loader reads three strided elements and quantises them.
#include <cuda_fp16.h>

#include <mutex>

#include "b2v_internal.h"

namespace b2v {

__device__ __forceinline__ int dp2a_lo(int coef, unsigned px, int acc) {
  int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(px), "r"(acc)); return d;
}
__device__ __forceinline__ int dp2a_hi(int coef, unsigned px, int acc) {
  int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(px), "r"(acc)); return d;
}
__device__ __forceinline__ uint4 ld_stream(const uint8_t* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_stream(uint8_t* p, unsigned v) {
  asm volatile("st.global.cs.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// pixel word: byte0 = B, byte1 = G, byte2 = R, byte3 = A (ignored: coefficient 0).  With S (RGBA, RGB) byte0 = R, byte2 = B.
__host__ __device__ constexpr int pack16(int lo, int hi) { return (int)(((unsigned)lo & 0xffffu) | ((unsigned)hi << 16)); }
// Colour matrices (14-bit coefficients).  0: BT.709 limited range, the H.264 path (DESIGN.md §3).  1: JFIF full-range BT.601, the
// JPEG stripe path (0.5 is coded as 8191 so that a saturated red / blue stays at 255; greys still give exactly 128) — the same
// numbers as oracle/csc_ref.c MATRIX[].
template <int M> struct Mx;
template <> struct Mx<0> { static constexpr int YR = KYR, YG = KYG, YB = KYB, UR = KUR, UG = KUG, UB = KUB, VR = KVR, VG = KVG, VB = KVB, YOFF = 16; };
template <> struct Mx<1> { static constexpr int YR = 4899, YG = 9617, YB = 1868, UR = -2765, UG = -5427, UB = 8191, VR = 8191, VG = -6860, VB = -1332, YOFF = 0; };
// Coefficients of bytes 0 and 2 of a pixel word, by channel order (S: byte 0 is R).
template <int M, bool S> struct Ord {
  using X = Mx<M>;
  static constexpr int Y0 = S ? X::YR : X::YB, Y2 = S ? X::YB : X::YR, U0 = S ? X::UR : X::UB, U2 = S ? X::UB : X::UR,
                       V0 = S ? X::VR : X::VB, V2 = S ? X::VB : X::VR;
};
// Rows of the general and scaled kernels, indexed by 2 * matrix + (pixel_format & 1): {Y, Cb, Cr coefficients of the channels
// read as (R, G, B)} and the luma offset.  The odd rows swap R and B: those kernels call byte 2 "R" and byte 0 "B" whatever
// the order, and the swapped row weighs each byte by its true channel, so the sums are the same integers.
__device__ const int c_mx[4][10] = {{KYR, KYG, KYB, KUR, KUG, KUB, KVR, KVG, KVB, 16}, {KYB, KYG, KYR, KUB, KUG, KUR, KVB, KVG, KVR, 16},
                                    {4899, 9617, 1868, -2765, -5427, 8191, 8191, -6860, -1332, 0},
                                    {1868, 9617, 4899, 8191, -5427, -2765, -1332, -6860, 8191, 0}};
constexpr int C_SEED = (128 << 16) + (1 << 15);

__device__ __forceinline__ unsigned dp2a_lo_u(unsigned coef, unsigned px, unsigned acc) {
  unsigned d; asm("dp2a.lo.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(px), "r"(acc)); return d;
}
__device__ __forceinline__ unsigned dp2a_hi_u(unsigned coef, unsigned px, unsigned acc) {
  unsigned d; asm("dp2a.hi.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(coef), "r"(px), "r"(acc)); return d;
}
// Luma with the coefficients scaled by 4 (all three are positive and 4*KYG still fits an UNSIGNED 16-bit dp2a lane):
// 4*(k.px) + 4*seed puts (k.px + seed) >> 14 into byte 2 of the accumulator, exactly (the factor 4 is exact), so the result is
// picked up by the same byte permute that packs four pixels — no shift instruction per pixel.  Chroma (>> 16) sits in byte 2 already.
template <int M, bool S>
__device__ __forceinline__ unsigned luma_b2(unsigned px) {      // Y in byte 2
  using X = Mx<M>;
  using O = Ord<M, S>;
  static_assert(4 * X::YG < 65536 && 4 * (X::YR + X::YG + X::YB) * 255 + 4 * ((X::YOFF << 14) + (1 << 13)) < (1 << 24), "luma accumulator must stay below byte 3");
  constexpr unsigned lo = (unsigned)pack16(4 * O::Y0, 4 * X::YG), hi = (unsigned)pack16(4 * O::Y2, 0), seed = 4u * (unsigned)((X::YOFF << 14) + (1 << 13));
  return dp2a_hi_u(hi, px, dp2a_lo_u(lo, px, seed));
}
__device__ __forceinline__ int chroma_acc(int clo, int chi, unsigned px, int acc) {
  return dp2a_hi(chi, px, dp2a_lo(clo, px, acc));
}
// byte 2 of each of four accumulators -> one word
__device__ __forceinline__ unsigned pack4_b2(unsigned a, unsigned b, unsigned c, unsigned d) {
  return __byte_perm(__byte_perm(a, b, 0x0062), __byte_perm(c, d, 0x0062), 0x5410);
}

// 4 px x 2 rows -> Y (two u32) + CbCr (one u32 = Cb0 Cr0 Cb1 Cr1)
template <int M, bool S>
__device__ __forceinline__ void convert_quad(const uint4& a, const uint4& b, unsigned& y0, unsigned& y1, unsigned& uv) {
  using X = Mx<M>;
  using O = Ord<M, S>;
  constexpr int CU_LO = pack16(O::U0, X::UG), CU_HI = pack16(O::U2, 0), CV_LO = pack16(O::V0, X::VG), CV_HI = pack16(O::V2, 0);
  y0 = pack4_b2(luma_b2<M, S>(a.x), luma_b2<M, S>(a.y), luma_b2<M, S>(a.z), luma_b2<M, S>(a.w));
  y1 = pack4_b2(luma_b2<M, S>(b.x), luma_b2<M, S>(b.y), luma_b2<M, S>(b.z), luma_b2<M, S>(b.w));
  int u0 = chroma_acc(CU_LO, CU_HI, b.y, chroma_acc(CU_LO, CU_HI, b.x, chroma_acc(CU_LO, CU_HI, a.y, chroma_acc(CU_LO, CU_HI, a.x, C_SEED))));
  int v0 = chroma_acc(CV_LO, CV_HI, b.y, chroma_acc(CV_LO, CV_HI, b.x, chroma_acc(CV_LO, CV_HI, a.y, chroma_acc(CV_LO, CV_HI, a.x, C_SEED))));
  int u1 = chroma_acc(CU_LO, CU_HI, b.w, chroma_acc(CU_LO, CU_HI, b.z, chroma_acc(CU_LO, CU_HI, a.w, chroma_acc(CU_LO, CU_HI, a.z, C_SEED))));
  int v1 = chroma_acc(CV_LO, CV_HI, b.w, chroma_acc(CV_LO, CV_HI, b.z, chroma_acc(CV_LO, CV_HI, a.w, chroma_acc(CV_LO, CV_HI, a.z, C_SEED))));
  uv = pack4_b2((unsigned)u0, (unsigned)v0, (unsigned)u1, (unsigned)v1);
}

// ---- fast path ---------------------------------------------------------------------------
// grid.x covers 4-px quads of a row, grid.y strides over groups of CSC_UNITS row pairs.
constexpr int CSC_UNITS = 2;     // units per thread (DESIGN.md §3)
constexpr int CSC_BLOCK = 160;   // threads per block, shrunk to a divisor of the row where one exists
template <int M, bool S>
__global__ void __launch_bounds__(256) csc_bgra_nv12_fast(CscParams p, int quads, int pairs) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (p.ts && threadIdx.x == 0) {   // device-side stopwatch of this launch: first block start .. last block end
    unsigned long long t0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0)); atomicMin(p.ts, t0);
  }
  const uint8_t* __restrict__ src = p.src + (size_t)(q < quads ? q : 0) * 16;
  if (q < quads)
  for (int pr0 = blockIdx.y * CSC_UNITS; pr0 < pairs; pr0 += gridDim.y * CSC_UNITS) {
    uint4 a[CSC_UNITS], b[CSC_UNITS];
#pragma unroll
    for (int u = 0; u < CSC_UNITS; u++) {
      int pr = pr0 + u;
      if (pr < pairs) {
        int r0 = min(2 * pr, p.src_h - 1), r1 = min(2 * pr + 1, p.src_h - 1);   // bottom padding rows replicate
        a[u] = ld_stream(src + (size_t)r0 * p.src_stride);
        b[u] = ld_stream(src + (size_t)r1 * p.src_stride);
      }
    }
#pragma unroll
    for (int u = 0; u < CSC_UNITS; u++) {
      int pr = pr0 + u;
      if (pr < pairs) {
        unsigned y0, y1, uv;
        convert_quad<M, S>(a[u], b[u], y0, y1, uv);
        st_stream(p.out_y + (size_t)(2 * pr) * p.coded_w + q * 4, y0);
        st_stream(p.out_y + (size_t)(2 * pr + 1) * p.coded_w + q * 4, y1);
        st_stream(p.out_uv + (size_t)pr * p.coded_w + q * 4, uv);
      }
    }
  }
  if (p.ts) {
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); atomicMax(p.ts + 1, t1); }
  }
}

// ---- packed 3-byte fast path (BGR / RGB, 1:1, width % 16 == 0, src and stride 16-byte aligned) --------------------------
// grid.x covers 16-px units of a row (C3_WARPS warps per block at most), grid.y strides over row pairs.  A warp's 32 units are
// 1536 B of a row: load k of lane l is the 16-byte chunk 32k + l (one contiguous 512 B per warp instruction); lane l then reads
// its chunks 3l .. 3l+2 back from shared memory (a 48-byte stride: the eight lanes of a quarter-warp cover 32 banks once).
constexpr int C3_WARPS = 8;
__device__ __forceinline__ void st_stream4(uint8_t* p, unsigned a, unsigned b, unsigned c, unsigned d) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// 12 bytes = 4 packed pixels -> 4 pixel words (bytes 0..2 = the pixel in memory order; byte 3 is left over and weighs 0)
__device__ __forceinline__ uint4 expand3(unsigned a, unsigned b, unsigned c) {
  return make_uint4(a, __byte_perm(a, b, 0x0543), __byte_perm(b, c, 0x0432), __byte_perm(c, c, 0x0321));
}
template <int M, bool S>
__global__ void __launch_bounds__(C3_WARPS * 32) csc_rgb24_nv12_fast(CscParams p, int units, int pairs) {
  __shared__ __align__(16) uint4 stage[C3_WARPS][2][96];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int u = blockIdx.x * blockDim.x + threadIdx.x, wu0 = u - lane;      // this thread's unit, the warp's first unit
  if (p.ts && threadIdx.x == 0) {
    unsigned long long t0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0)); atomicMin(p.ts, t0);
  }
  if (wu0 < units) {                                                         // warp-uniform
    const int chunks = min(96, 3 * (units - wu0));
    for (int pr = blockIdx.y; pr < pairs; pr += gridDim.y) {
      const int r0 = min(2 * pr, p.src_h - 1), r1 = min(2 * pr + 1, p.src_h - 1);   // bottom padding rows replicate
      const uint8_t* g0 = p.src + (size_t)r0 * p.src_stride + (size_t)wu0 * 48;
      const uint8_t* g1 = p.src + (size_t)r1 * p.src_stride + (size_t)wu0 * 48;
      uint4 a[3], b[3];
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const int c = 32 * k + lane;
        if (c < chunks) { a[k] = ld_stream(g0 + 16 * c); b[k] = ld_stream(g1 + 16 * c); }
      }
      __syncwarp();                                   // the previous pair's reads of `stage` are done
#pragma unroll
      for (int k = 0; k < 3; k++) {
        const int c = 32 * k + lane;
        if (c < chunks) { stage[w][0][c] = a[k]; stage[w][1][c] = b[k]; }
      }
      __syncwarp();
      if (u < units) {
        const uint4 x0 = stage[w][0][3 * lane], x1 = stage[w][0][3 * lane + 1], x2 = stage[w][0][3 * lane + 2];
        const uint4 z0 = stage[w][1][3 * lane], z1 = stage[w][1][3 * lane + 1], z2 = stage[w][1][3 * lane + 2];
        unsigned y0[4], y1[4], uv[4];
        convert_quad<M, S>(expand3(x0.x, x0.y, x0.z), expand3(z0.x, z0.y, z0.z), y0[0], y1[0], uv[0]);
        convert_quad<M, S>(expand3(x0.w, x1.x, x1.y), expand3(z0.w, z1.x, z1.y), y0[1], y1[1], uv[1]);
        convert_quad<M, S>(expand3(x1.z, x1.w, x2.x), expand3(z1.z, z1.w, z2.x), y0[2], y1[2], uv[2]);
        convert_quad<M, S>(expand3(x2.y, x2.z, x2.w), expand3(z2.y, z2.z, z2.w), y0[3], y1[3], uv[3]);
        st_stream4(p.out_y + (size_t)(2 * pr) * p.coded_w + u * 16, y0[0], y0[1], y0[2], y0[3]);
        st_stream4(p.out_y + (size_t)(2 * pr + 1) * p.coded_w + u * 16, y1[0], y1[1], y1[2], y1[3]);
        st_stream4(p.out_uv + (size_t)pr * p.coded_w + u * 16, uv[0], uv[1], uv[2], uv[3]);
      }
    }
  }
  if (p.ts) {
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); atomicMax(p.ts + 1, t1); }
  }
}

// ---- planar 1:1 fast path (three planes of B2V_DT_* elements; rows contiguous; planes, row stride and outputs 16-byte aligned) ----
// element -> 8-bit sample (DESIGN.md §3): rint_half_even(255 * min(max(x, 0), 1)), one fp32 multiplication; __saturatef(NaN) is 0
__device__ __forceinline__ unsigned quant(float x) { return (unsigned)__float2int_rn(__saturatef(x) * 255.0f); }
__device__ __forceinline__ unsigned quant_h2(unsigned two) {            // two fp16 -> samples in bytes 0 and 1
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&two));
  return quant(f.x) | (quant(f.y) << 8);
}
__device__ __forceinline__ unsigned quant_b2(unsigned two) {            // two bf16: each is the high half of its fp32
  return quant(__uint_as_float(two << 16)) | (quant(__uint_as_float(two & 0xffff0000u)) << 8);
}
__host__ __device__ constexpr int planar_px(int dt) { return dt == B2V_DT_U8 ? 16 : dt == B2V_DT_F32 ? 4 : 8; }   // elements of one 16-byte load
// one 16-byte load -> its samples, four to a word
template <int DT>
__device__ __forceinline__ void quant16(const uint4& v, unsigned (&w)[planar_px(DT) / 4]) {
  if constexpr (DT == B2V_DT_U8) { w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w; }
  else if constexpr (DT == B2V_DT_F16) { w[0] = quant_h2(v.x) | (quant_h2(v.y) << 16); w[1] = quant_h2(v.z) | (quant_h2(v.w) << 16); }
  else if constexpr (DT == B2V_DT_BF16) { w[0] = quant_b2(v.x) | (quant_b2(v.y) << 16); w[1] = quant_b2(v.z) | (quant_b2(v.w) << 16); }
  else w[0] = quant(__uint_as_float(v.x)) | (quant(__uint_as_float(v.y)) << 8) | (quant(__uint_as_float(v.z)) << 16) | (quant(__uint_as_float(v.w)) << 24);
}
// four samples of each plane -> four pixel words (byte 0 = B, 1 = G, 2 = R; byte 3 is left over and weighs 0)
__device__ __forceinline__ uint4 weave(unsigned b, unsigned g, unsigned r) {
  const unsigned bg01 = __byte_perm(b, g, 0x5140), bg23 = __byte_perm(b, g, 0x7362);
  return make_uint4(__byte_perm(bg01, r, 0x4410), __byte_perm(bg01, r, 0x5532), __byte_perm(bg23, r, 0x6610), __byte_perm(bg23, r, 0x7732));
}
template <int Q>
__device__ __forceinline__ void st_words(uint8_t* p, const unsigned (&w)[Q]) {
  if constexpr (Q == 4) st_stream4(p, w[0], w[1], w[2], w[3]);
  else if constexpr (Q == 2) asm volatile("st.global.cs.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(w[0]), "r"(w[1]) : "memory");
  else st_stream(p, w[0]);
}
// p.src is the blue plane, pg and pr the green and red ones.  grid.x covers the units (one 16-byte load wide) of a row, grid.y
// strides over row pairs.
template <int M, int DT>
__global__ void __launch_bounds__(256) csc_planar_nv12_fast(CscParams p, const uint8_t* __restrict__ pg, const uint8_t* __restrict__ pr, int units, int pairs) {
  constexpr int PX = planar_px(DT), Q = PX / 4;
  const int u = blockIdx.x * blockDim.x + threadIdx.x;
  if (p.ts && threadIdx.x == 0) {
    unsigned long long t0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0)); atomicMin(p.ts, t0);
  }
  if (u < units)
  for (int pair = blockIdx.y; pair < pairs; pair += gridDim.y) {
    const int r0 = min(2 * pair, p.src_h - 1), r1 = min(2 * pair + 1, p.src_h - 1);   // bottom padding rows replicate
    const size_t o0 = (size_t)r0 * p.src_stride + (size_t)u * 16, o1 = (size_t)r1 * p.src_stride + (size_t)u * 16;
    const uint4 vb0 = ld_stream(p.src + o0), vg0 = ld_stream(pg + o0), vr0 = ld_stream(pr + o0);
    const uint4 vb1 = ld_stream(p.src + o1), vg1 = ld_stream(pg + o1), vr1 = ld_stream(pr + o1);
    unsigned b0[Q], g0[Q], c0[Q], b1[Q], g1[Q], c1[Q], y0[Q], y1[Q], uv[Q];
    quant16<DT>(vb0, b0); quant16<DT>(vg0, g0); quant16<DT>(vr0, c0);
    quant16<DT>(vb1, b1); quant16<DT>(vg1, g1); quant16<DT>(vr1, c1);
#pragma unroll
    for (int k = 0; k < Q; k++) convert_quad<M, false>(weave(b0[k], g0[k], c0[k]), weave(b1[k], g1[k], c1[k]), y0[k], y1[k], uv[k]);
    st_words<Q>(p.out_y + (size_t)(2 * pair) * p.coded_w + u * PX, y0);
    st_words<Q>(p.out_y + (size_t)(2 * pair + 1) * p.coded_w + u * PX, y1);
    st_words<Q>(p.out_uv + (size_t)pair * p.coded_w + u * PX, uv);
  }
  if (p.ts) {
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); atomicMax(p.ts + 1, t1); }
  }
}

// ---- general path: bilinear scale and/or ragged width, one thread per 2x2 output block -----
__device__ __forceinline__ unsigned load_elem(const uint8_t* e, int dtype) {
  switch (dtype) {
    case B2V_DT_U8: return *e;
    case B2V_DT_F16: return quant(__half2float(*reinterpret_cast<const __half*>(e)));
    case B2V_DT_BF16: return quant(__uint_as_float((unsigned)*reinterpret_cast<const uint16_t*>(e) << 16));
    default: return quant(*reinterpret_cast<const float*>(e));
  }
}
// pixel word of pixel x of a row: bytes 0..2 are its colour bytes in memory order (3-byte formats: any alignment), or the
// quantised elements of channels 0..2 of a tensor, wherever its strides put them
__device__ __forceinline__ unsigned load_px(const uint8_t* row, int x, const CscSource& p) {
  if (p.stride_c == 0) {
    if (p.fmt < B2V_PIX_BGR) return *(const unsigned*)(row + x * 4);
    const uint8_t* q = row + x * 3;
    return (unsigned)q[0] | ((unsigned)q[1] << 8) | ((unsigned)q[2] << 16);
  }
  const uint8_t* e = row + (size_t)x * p.stride_x;
  return load_elem(e, p.dtype) | (load_elem(e + p.stride_c, p.dtype) << 8) | (load_elem(e + 2 * p.stride_c, p.dtype) << 16);
}
// B = byte 0, R = byte 2 of the pixel word: swapped for RGBA / RGB, which the matrix row c_mx[2 * matrix + 1] accounts for
__device__ __forceinline__ void fetch_bgr(const CscSource& p, int x, int y, int& B, int& G, int& R) {
  int x0, x1, fx, y0, y1, fy;
  if (p.tx) { Tap t = p.tx[x]; x0 = t.i0; x1 = t.i1; fx = t.f; } else { x0 = x1 = x; fx = 0; }
  if (p.ty) { Tap t = p.ty[y]; y0 = t.i0; y1 = t.i1; fy = t.f; } else { y0 = y1 = y; fy = 0; }
  const uint8_t* r0 = p.src + (size_t)y0 * p.src_stride;
  const uint8_t* r1 = p.src + (size_t)y1 * p.src_stride;
  unsigned p00 = load_px(r0, x0, p);
  if (fx == 0 && fy == 0) { B = p00 & 255; G = (p00 >> 8) & 255; R = (p00 >> 16) & 255; return; }
  unsigned p01 = load_px(r0, x1, p), p10 = load_px(r1, x0, p), p11 = load_px(r1, x1, p);
  int out[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    int s = 8 * c;
    int top = (int)((p00 >> s) & 255) * (256 - fx) + (int)((p01 >> s) & 255) * fx;
    int bot = (int)((p10 >> s) & 255) * (256 - fx) + (int)((p11 >> s) & 255) * fx;
    out[c] = (top * (256 - fy) + bot * fy + (1 << 15)) >> 16;
  }
  B = out[0]; G = out[1]; R = out[2];
}

__global__ void __launch_bounds__(256) csc_bgra_nv12_general(CscSource p) {
  int bx = blockIdx.x * blockDim.x + threadIdx.x;   // 2x2 block column
  int by = blockIdx.y * blockDim.y + threadIdx.y;
  if (bx * 2 >= p.coded_w || by * 2 >= p.coded_h) return;
  const int* mx = c_mx[2 * p.matrix + (p.fmt & 1)];
  int sb = 0, sg = 0, sr = 0;
  unsigned yy[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    int x = min(bx * 2 + (k & 1), p.dst_w - 1), y = min(by * 2 + (k >> 1), p.dst_h - 1);
    int B, G, R;
    fetch_bgr(p, x, y, B, G, R);
    yy[k] = (unsigned)(mx[0] * R + mx[1] * G + mx[2] * B + (mx[9] << 14) + (1 << 13)) >> 14;
    sb += B; sg += G; sr += R;
  }
  unsigned cb = (unsigned)(mx[3] * sr + mx[4] * sg + mx[5] * sb + C_SEED) >> 16;
  unsigned cr = (unsigned)(mx[6] * sr + mx[7] * sg + mx[8] * sb + C_SEED) >> 16;
  *(uint16_t*)(p.out_y + (size_t)(by * 2) * p.coded_w + bx * 2) = (uint16_t)(yy[0] | (yy[1] << 8));
  *(uint16_t*)(p.out_y + (size_t)(by * 2 + 1) * p.coded_w + bx * 2) = (uint16_t)(yy[2] | (yy[3] << 8));
  *(uint16_t*)(p.out_uv + (size_t)by * p.coded_w + bx * 2) = (uint16_t)(cb | (cr << 8));
}

// ---- scaled path: fused bilinear scale + CSC through a shared-memory tile -----------------------------------------------------
// One CTA produces SC_TW x SC_TH output pixels (one thread per 2x2 block: the chroma sample needs all four).  The source
// footprint of the tile — tx[first].i0 .. tx[last].i1 by ty[first].i0 .. ty[last].i1, a few KB whatever the scale factor — is
// staged in shared memory with 16-byte loads; every tap is then a shared-memory read.  The arithmetic is the spec's (oracle/
// csc_ref.c fetch_bgr): per channel top/bottom horizontal blends at full precision (B and R ride in the two 16-bit halves of one
// word: 255*256 fits), one vertical blend, one rounding.  Roofline: 4 B per source pixel read + 1.5 B per output pixel written.
// Packed 3-byte sources and tensors are staged as the same pixel words (any alignment, quantised once), so everything after the
// staging is shared.
constexpr int SC_TW = 64, SC_TH = 8, SC_THREADS = (SC_TW / 2) * (SC_TH / 2);

__device__ __forceinline__ void blend_px(const uint32_t* r0, const uint32_t* r1, int x0, int x1, int fx, int fy, int& B, int& G, int& R) {
  const uint32_t p00 = r0[x0], p01 = r0[x1], p10 = r1[x0], p11 = r1[x1];
  const uint32_t M = 0x00ff00ffu;
  const uint32_t wx1 = (uint32_t)fx, wx0 = 256u - wx1;
  const uint32_t tbr = (p00 & M) * wx0 + (p01 & M) * wx1, bbr = (p10 & M) * wx0 + (p11 & M) * wx1;        // [B | R << 16], each <= 65280
  const uint32_t tg = ((p00 >> 8) & 255u) * wx0 + ((p01 >> 8) & 255u) * wx1, bg = ((p10 >> 8) & 255u) * wx0 + ((p11 >> 8) & 255u) * wx1;
  const uint32_t wy1 = (uint32_t)fy, wy0 = 256u - wy1;
  B = (int)(((tbr & 0xffffu) * wy0 + (bbr & 0xffffu) * wy1 + (1u << 15)) >> 16);
  R = (int)(((tbr >> 16) * wy0 + (bbr >> 16) * wy1 + (1u << 15)) >> 16);
  G = (int)((tg * wy0 + bg * wy1 + (1u << 15)) >> 16);
}

__global__ void __launch_bounds__(SC_THREADS) csc_bgra_nv12_scaled(CscSource p, int fw_cap, int fh_cap) {
  extern __shared__ __align__(16) uint32_t sc_tile[];            // fh_cap rows of fw_cap pixels (fw_cap % 4 == 0)
  const int tid = threadIdx.x;
  const int ox0 = blockIdx.x * SC_TW, oy0 = blockIdx.y * SC_TH;
  // footprint of this tile in the source (output coordinates beyond the visible picture replicate its last row / column)
  const int xf = min(ox0, p.dst_w - 1), xl = min(ox0 + SC_TW - 1, p.dst_w - 1);
  const int yf = min(oy0, p.dst_h - 1), yl = min(oy0 + SC_TH - 1, p.dst_h - 1);
  const int xs0 = p.tx[xf].i0 & ~3, xs1 = p.tx[xl].i1, ys0 = p.ty[yf].i0, ys1 = p.ty[yl].i1;
  const int fw4 = (xs1 - xs0 + 4) >> 2, fh = ys1 - ys0 + 1;      // quads per row, rows
  for (int i = tid; i < fh * fw4; i += SC_THREADS) {
    const int r = i / fw4, c = i - r * fw4, sx = xs0 + 4 * c;
    const uint8_t* row = p.src + (size_t)(ys0 + r) * p.src_stride;
    uint4 v;
    if (sx + 3 < p.src_w && p.stride_c == 0 && p.fmt < B2V_PIX_BGR) v = ld_stream(row + (size_t)sx * 4);
    else {                          // packed 3-byte pixels, a tensor's elements, or the last quad of a row whose width is not a multiple of 4
      v.x = load_px(row, sx, p);
      v.y = sx + 1 < p.src_w ? load_px(row, sx + 1, p) : 0u;
      v.z = sx + 2 < p.src_w ? load_px(row, sx + 2, p) : 0u;
      v.w = sx + 3 < p.src_w ? load_px(row, sx + 3, p) : 0u;
    }
    *reinterpret_cast<uint4*>(&sc_tile[r * fw_cap + 4 * c]) = v;
  }
  (void)fh_cap;
  __syncthreads();
  const int bx = tid % (SC_TW / 2), by = tid / (SC_TW / 2);
  const int ox = ox0 + 2 * bx, oy = oy0 + 2 * by;
  if (ox >= p.coded_w || oy >= p.coded_h) return;
  const int* mx = c_mx[2 * p.matrix + (p.fmt & 1)];
  int sb = 0, sg = 0, sr = 0;
  unsigned yy[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int x = min(ox + (k & 1), p.dst_w - 1), y = min(oy + (k >> 1), p.dst_h - 1);
    const Tap ax = p.tx[x], ay = p.ty[y];
    int B, G, R;
    blend_px(&sc_tile[(ay.i0 - ys0) * fw_cap], &sc_tile[(ay.i1 - ys0) * fw_cap], ax.i0 - xs0, ax.i1 - xs0, ax.f, ay.f, B, G, R);
    yy[k] = (unsigned)(mx[0] * R + mx[1] * G + mx[2] * B + (mx[9] << 14) + (1 << 13)) >> 14;
    sb += B; sg += G; sr += R;
  }
  const unsigned cb = (unsigned)(mx[3] * sr + mx[4] * sg + mx[5] * sb + C_SEED) >> 16;
  const unsigned cr = (unsigned)(mx[6] * sr + mx[7] * sg + mx[8] * sb + C_SEED) >> 16;
  *reinterpret_cast<uint16_t*>(p.out_y + (size_t)oy * p.coded_w + ox) = (uint16_t)(yy[0] | (yy[1] << 8));
  *reinterpret_cast<uint16_t*>(p.out_y + (size_t)(oy + 1) * p.coded_w + ox) = (uint16_t)(yy[2] | (yy[3] << 8));
  *reinterpret_cast<uint16_t*>(p.out_uv + (size_t)(oy >> 1) * p.coded_w + ox) = (uint16_t)(cb | (cr << 8));
}

// host side ---------------------------------------------------------------------------------
void make_taps_host(Tap* t, int dn, int sn) {
  for (int d = 0; d < dn; d++) {
    if (dn == sn) { t[d] = Tap{d, d, 0, 0}; continue; }
    int64_t pos = (((int64_t)(2 * d + 1) * sn) << 15) / dn - (1 << 15);
    int64_t hi = (int64_t)(sn - 1) << 16;
    if (pos < 0) pos = 0;
    if (pos > hi) pos = hi;
    int i0 = (int)(pos >> 16);
    t[d] = Tap{i0, i0 + 1 < sn ? i0 + 1 : sn - 1, (int)((pos >> 8) & 255), 0};
  }
}

// Opt-in dynamic shared memory above 48 KB.  cudaFuncSetAttribute applies to the CURRENT device only, so the size already
// granted is remembered per device (a session on a second GPU needs its own call), and submitters of several sessions may
// get here at once: the record is guarded.
constexpr int kAttrDevices = 64;
static std::mutex g_attr_mu;
static int g_attr_scaled[kAttrDevices];
static void opt_in_smem(const void* fn, int* granted, int smem) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_attr_mu);
  if (dev >= 0 && dev < kAttrDevices && smem <= granted[dev]) return;
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess && dev >= 0 && dev < kAttrDevices) granted[dev] = smem;
}

template <int M>
static void launch_planar(const CscSource& p, const uint8_t* pg, const uint8_t* pr, dim3 grid, int block, int units, int pairs, cudaStream_t st) {
  switch (p.dtype) {
    case B2V_DT_U8: csc_planar_nv12_fast<M, B2V_DT_U8><<<grid, block, 0, st>>>(p, pg, pr, units, pairs); break;
    case B2V_DT_F16: csc_planar_nv12_fast<M, B2V_DT_F16><<<grid, block, 0, st>>>(p, pg, pr, units, pairs); break;
    case B2V_DT_BF16: csc_planar_nv12_fast<M, B2V_DT_BF16><<<grid, block, 0, st>>>(p, pg, pr, units, pairs); break;
    default: csc_planar_nv12_fast<M, B2V_DT_F32><<<grid, block, 0, st>>>(p, pg, pr, units, pairs); break;
  }
}

int launch_csc(const CscSource& p, cudaStream_t st) {
  const bool tensor = p.stride_c != 0, swap = (p.fmt & 1) != 0, packed3 = p.fmt >= B2V_PIX_BGR;
  const bool one_to_one = p.tx == nullptr && p.ty == nullptr && p.dst_w == p.src_w && p.dst_h == p.src_h && p.coded_w == p.dst_w;
  const bool aligned16 = (p.src_stride % 16) == 0 && ((uintptr_t)p.src % 16) == 0;
  const bool fast = !tensor && one_to_one && !packed3 && (p.coded_w % 4) == 0 && aligned16 && ((uintptr_t)p.out_y % 4) == 0 && ((uintptr_t)p.out_uv % 4) == 0;
  const bool fast3 = !tensor && one_to_one && packed3 && (p.coded_w % 16) == 0 && aligned16 && ((uintptr_t)p.out_y % 16) == 0 && ((uintptr_t)p.out_uv % 16) == 0;
  const int ppx = planar_px(p.dtype), elem = 16 / ppx;       // pixels per 16-byte load of a plane, bytes per element
  const bool planar = tensor && one_to_one && p.stride_x == elem && aligned16 && (p.stride_c % 16) == 0 && (p.coded_w % ppx) == 0 &&
                      ((uintptr_t)p.out_y % ppx) == 0 && ((uintptr_t)p.out_uv % ppx) == 0;
  if (planar) {
    const int units = p.coded_w / ppx, pairs = p.coded_h / 2;
    int block = 256;                                           // the block that leaves the fewest idle threads in a row of units
    for (int b = 224; b >= 64; b -= 32)
      if ((units + b - 1) / b * b < (units + block - 1) / block * block) block = b;
    const dim3 grid((units + block - 1) / block, pairs < 65535 ? pairs : 65535);
    // channel order: which plane feeds which byte of the pixel word.  The kernel's p.src is the blue plane.
    CscSource q = p;
    q.src = p.src + (swap ? 2 * p.stride_c : 0);
    const uint8_t* pg = p.src + p.stride_c;
    const uint8_t* pr = p.src + (swap ? 0 : 2 * p.stride_c);
    if (p.matrix == 1) launch_planar<1>(q, pg, pr, grid, block, units, pairs, st);
    else launch_planar<0>(q, pg, pr, grid, block, units, pairs, st);
  } else if (fast) {
    const int quads = p.coded_w / 4, pairs = p.coded_h / 2;
    int block = CSC_BLOCK;
    while (block > 64 && quads % block != 0) block -= 32;   // prefer a divisor of the row
    if (quads % block != 0) block = CSC_BLOCK;
    int gy = (pairs + CSC_UNITS - 1) / CSC_UNITS;            // one group of CSC_UNITS row pairs per block
    if (gy > 65535) gy = 65535;
    const dim3 grid((quads + block - 1) / block, gy);
    if (p.matrix == 1) {
      if (swap) csc_bgra_nv12_fast<1, true><<<grid, block, 0, st>>>(p, quads, pairs);
      else csc_bgra_nv12_fast<1, false><<<grid, block, 0, st>>>(p, quads, pairs);
    } else {
      if (swap) csc_bgra_nv12_fast<0, true><<<grid, block, 0, st>>>(p, quads, pairs);
      else csc_bgra_nv12_fast<0, false><<<grid, block, 0, st>>>(p, quads, pairs);
    }
  } else if (fast3) {
    // whole warps of 16-px units, spread evenly over as few blocks of at most C3_WARPS warps as the row needs
    const int units = p.coded_w / 16, pairs = p.coded_h / 2;
    const int warps = (units + 31) / 32, bx = (warps + C3_WARPS - 1) / C3_WARPS, block = 32 * ((warps + bx - 1) / bx);
    const dim3 grid(bx, pairs < 65535 ? pairs : 65535);
    if (p.matrix == 1) {
      if (swap) csc_rgb24_nv12_fast<1, true><<<grid, block, 0, st>>>(p, units, pairs);
      else csc_rgb24_nv12_fast<1, false><<<grid, block, 0, st>>>(p, units, pairs);
    } else {
      if (swap) csc_rgb24_nv12_fast<0, true><<<grid, block, 0, st>>>(p, units, pairs);
      else csc_rgb24_nv12_fast<0, false><<<grid, block, 0, st>>>(p, units, pairs);
    }
  } else {
    // scaled: the tiled kernel when the tile's source footprint fits shared memory (any sane scale factor), else the general one.
    // 4-byte pixels are staged with 16-byte loads, so they need a 16-byte aligned source; 3-byte pixels are read bytewise and a
    // tensor element by element.
    if (p.tx && p.ty && (tensor || packed3 || aligned16)) {
      const long long fw = ((long long)SC_TW * p.src_w + p.dst_w - 1) / p.dst_w + 8, fh = ((long long)SC_TH * p.src_h + p.dst_h - 1) / p.dst_h + 3;
      const int fw_cap = (int)((fw + 3) & ~3LL), fh_cap = (int)fh;
      const long long smem = (long long)fw_cap * fh_cap * 4;
      if (smem <= 96 * 1024) {
        if (smem > 48 * 1024) opt_in_smem((const void*)csc_bgra_nv12_scaled, g_attr_scaled, (int)smem);
        dim3 grid((p.coded_w + SC_TW - 1) / SC_TW, (p.coded_h + SC_TH - 1) / SC_TH);
        csc_bgra_nv12_scaled<<<grid, SC_THREADS, (size_t)smem, st>>>(p, fw_cap, fh_cap);
        return 1;
      }
    }
    dim3 block(32, 8);
    dim3 grid((p.coded_w / 2 + 31) / 32, (p.coded_h / 2 + 7) / 8);
    csc_bgra_nv12_general<<<grid, block, 0, st>>>(p);
  }
  return 1;
}

}  // namespace b2v
