// quality.cu — k_quality: per-band SSE (Y, Cb, Cr) and SSIM of the coded picture S against its reconstruction R
// (B2V_FLAG_QUALITY; definition in DESIGN.md §5.11 and include/b2video.h).
//
// One warp walks a strip of 31 owned 4x4 luma blocks (124 columns, plus one halo block column on lane 31) down SEG block rows
// (plus one halo block row).  Every step loads one 4x4 block of S and R per lane (and the two NV12 chroma rows under it), takes
// its four sums with dp4a, and forms the 8x8 window whose origin is the block above from the 2x2 blocks around it: the column
// pair through the lane's own registers, the row pair through one shuffle.  So each sample is read once (the halos add 1/31 and
// 1/SEG) and no 64-sample sum is ever recomputed.  SSEs accumulate as exact integers, SSIM as round(ssim * 2^40) in int64, so
// the result does not depend on the order of the atomics.  A block sums its warps in shared memory per band, adds to the global
// accumulators, and the last block to finish copies them into the access unit's quality table and zeroes them for the next
// picture: one launch, no memset.
#include "b2v_internal.h"

namespace b2v {

namespace {

constexpr int QW = 4;                      // warps per block: consecutive segments of one strip
constexpr int SEG = 8;                     // block rows (4 luma rows each) a warp owns
constexpr int KB = 4 * SEG * QW / 16 + 1;  // bands a block's rows can touch (bands are whole macroblock rows)
constexpr int NF = 5;                      // fields of a QualityEntry
constexpr double kQ40 = 1099511627776.0;   // 2^40

struct Acc {
  unsigned int sse[3] = {0, 0, 0};
  long long ssim = 0;
  int windows = 0;
};

__device__ __forceinline__ unsigned ld4(const uint8_t* p) { return __ldg(reinterpret_cast<const unsigned*>(p)); }

// warp sum of `a` into the block's shared record of `band`
__device__ __forceinline__ void flush(Acc& a, unsigned long long (*sh)[NF], int band, int band_lo) {
  unsigned long long v[NF] = {a.sse[0], a.sse[1], a.sse[2], (unsigned long long)a.ssim, (unsigned long long)a.windows};
#pragma unroll
  for (int i = 0; i < NF; i++)
    for (int o = 16; o; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int i = 0; i < NF; i++)
      if (v[i]) atomicAdd(&sh[band - band_lo][i], v[i]);
  a = Acc{};
}

}  // namespace

__global__ void __launch_bounds__(32 * QW) k_quality(QualityParams p, int blocks_per_strip, int n_seg) {
  __shared__ unsigned long long sh[KB][NF];
  __shared__ bool s_last;
  const int tid = threadIdx.x, lane = tid & 31;
  for (int i = tid; i < KB * NF; i += blockDim.x) sh[i / NF][i % NF] = 0;
  const int strip = blockIdx.x / blocks_per_strip, seg0 = (blockIdx.x % blocks_per_strip) * QW;
  const int band_lo = 4 * SEG * seg0 / p.band_px;
  __syncthreads();

  const int seg = seg0 + (tid >> 5);
  if (seg < n_seg) {
    const int x = 4 * (strip * 31 + lane);
    const bool col_in = x < p.coded_w;
    // bytes counted by the SSEs: the visible ones (dst_w is even) of an owned block (lane 31 is the next strip's lane 0)
    const unsigned vis = lane == 31 ? 0u : x + 4 <= p.dst_w ? 0xffffffffu : x + 2 <= p.dst_w ? 0x0000ffffu : 0u;
    const bool win_col = lane < 31 && x + 8 <= p.dst_w;
    const size_t plane = (size_t)p.coded_w * p.coded_h;
    int band = 4 * SEG * seg / p.band_px;
    Acc a;
    unsigned psx = 0, psy = 0, pq = 0, pp = 0;     // sums of the block above
    for (int k = 0; k <= SEG; k++) {
      const int y = 4 * (SEG * seg + k);
      if (y >= p.dst_h) break;
      unsigned s[4] = {0, 0, 0, 0}, r[4] = {0, 0, 0, 0};
      if (col_in) {
#pragma unroll
        for (int i = 0; i < 4; i++) {
          const size_t o = (size_t)(y + i) * p.coded_w + x;
          s[i] = ld4(p.src + o); r[i] = ld4(p.recon + o);
        }
      }
      unsigned bsx = 0, bsy = 0, bq = 0, bp = 0;
#pragma unroll
      for (int i = 0; i < 4; i++) {
        bsx = __dp4a(s[i], 0x01010101u, bsx); bsy = __dp4a(r[i], 0x01010101u, bsy);
        bq = __dp4a(s[i], s[i], bq); bq = __dp4a(r[i], r[i], bq); bp = __dp4a(s[i], r[i], bp);
      }
      if (k > 0) {                                  // the window with origin (x, y - 4): blocks (x, y - 4), (x + 4, y - 4), (x, y), (x + 4, y)
        unsigned wsx = psx + bsx, wsy = psy + bsy, wq = pq + bq, wp = pp + bp;
        wsx += __shfl_down_sync(0xffffffffu, wsx, 1); wsy += __shfl_down_sync(0xffffffffu, wsy, 1);
        wq += __shfl_down_sync(0xffffffffu, wq, 1); wp += __shfl_down_sync(0xffffffffu, wp, 1);
        if (win_col && y + 4 <= min(p.dst_h, (band + 1) * p.band_px)) {      // wholly inside the band of its origin row
          const long long Sx = wsx, Sy = wsy;
          const long long V = 64LL * wq - Sx * Sx - Sy * Sy, C = 64LL * wp - Sx * Sy;
          const double num = __dmul_rn((double)(2 * Sx * Sy + 416), (double)(2 * C + 235963));
          const double den = __dmul_rn((double)(Sx * Sx + Sy * Sy + 416), (double)(V + 235963));
          a.ssim += __double2ll_rn(__ddiv_rn(num, den) * kQ40);
          a.windows++;
        }
      }
      if (k == SEG) break;                          // the halo row: its samples belong to the next segment
      if (y / p.band_px != band) { flush(a, sh, band, band_lo); band = y / p.band_px; }
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const unsigned d = __vabsdiffu4(s[i], r[i]) & vis;
        if (y + i < p.dst_h) a.sse[0] = __dp4a(d, d, a.sse[0]);
      }
      if (col_in) {
#pragma unroll
        for (int j = 0; j < 2; j++) {               // NV12 chroma rows 2 * (y / 4) + j: Cb in the even bytes, Cr in the odd
          const int cy = y / 2 + j;
          if (2 * cy >= p.dst_h) continue;
          const size_t o = plane + (size_t)cy * p.coded_w + x;
          const unsigned d = __vabsdiffu4(ld4(p.src + o), ld4(p.recon + o)) & vis;
          a.sse[1] = __dp4a(d & 0x00ff00ffu, d, a.sse[1]);
          a.sse[2] = __dp4a(d & 0xff00ff00u, d, a.sse[2]);
        }
      }
      psx = bsx; psy = bsy; pq = bq; pp = bp;
    }
    flush(a, sh, band, band_lo);
  }
  __syncthreads();

  unsigned long long* acc = reinterpret_cast<unsigned long long*>(p.acc);
  for (int i = tid; i < KB * NF; i += blockDim.x) {
    const int b = band_lo + i / NF;
    if (b < p.n_bands && sh[i / NF][i % NF]) atomicAdd(&acc[b * NF + i % NF], sh[i / NF][i % NF]);
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(p.done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  unsigned long long* out = reinterpret_cast<unsigned long long*>(p.out);
  for (int i = tid; i < p.n_bands * NF; i += blockDim.x) out[i] = atomicExch(&acc[i], 0ULL);
  if (tid == 0) *p.done = 0;
}

int launch_quality(const QualityParams& p, cudaStream_t st) {
  const int strips = ((p.dst_w + 3) / 4 + 30) / 31;
  const int n_seg = ((p.dst_h + 3) / 4 + SEG - 1) / SEG;
  const int bps = (n_seg + QW - 1) / QW;
  k_quality<<<strips * bps, 32 * QW, 0, st>>>(p, bps, n_seg);
  return 1;
}

}  // namespace b2v
