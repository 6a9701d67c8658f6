// h264_cap.cu — B2V_FLAG_SIZE_CAP: a P picture whose macroblock layer exceeds the caller's byte budget is coded once more at a
// coarser QP, decided on the GPU with no host round trip (DESIGN.md §5.15; CPU restatement: oracle/h264_cap_ref.c).
//   k_cavlc_mb (the count) -> k_size_cap -> k_requant -> k_cavlc_recode, then the slice build and the pack as for every picture.
// k_size_cap is one block: it sums the macroblocks' CAVLC bit counts and applies the rule (include/b2video.h).  k_requant
// (h264_inter.cu) and k_cavlc_recode (h264_entropy.cu) return at once when it did not recode the picture.
#include "h264_common.cuh"
#include "h264_encoder.h"
#include "h264_kernels.h"

namespace b2v {

constexpr int CAP_THREADS = 1024;
constexpr int PCM_SAMPLE_BITS = 384 * 8;      // pcm_sample_luma + pcm_sample_chroma of an I_PCM macroblock (7.3.5)

__global__ void __launch_bounds__(CAP_THREADS) k_size_cap(FrameCtx f) {
  __shared__ unsigned long long s_sum[CAP_THREADS / 32];
  const int mbs = f.mbw * f.mbh, tid = threadIdx.x;
  unsigned long long bits = 0;
  // a P_Skip macroblock counts 0; an I_PCM macroblock its mb_type and its 384 samples (its alignment bits are not counted)
  for (int i = tid; i < mbs; i += CAP_THREADS) {
    const uint32_t v = f.mb_nbits[i];
    bits += (v & 0x3fffffffu) + ((v >> 30) == 1u ? PCM_SAMPLE_BITS : 0u);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) bits += __shfl_xor_sync(FULL, bits, d);
  if ((tid & 31) == 0) s_sum[tid >> 5] = bits;
  __syncthreads();
  if (tid != 0) return;
  long long total = 0;
  for (int w = 0; w < CAP_THREADS / 32; w++) total += (long long)s_sum[w];
  const int par = f.pic & 1, qp = frame_qp(f);
  const bool cut = f.scut && f.scut->cut[par];      // a cut picture is an intra picture: not capped
  const long long cap_bits = 8LL * f.cap_bytes;
  int q = qp;
  if (f.cap_bytes > 0 && !cut && qp < 51 && (total + 7) / 8 > f.cap_bytes) {
    int d = 1;
    while (d < 51 - qp && total > (cap_bits * cap_t[d]) >> 16) d++;
    q = qp + d;
  }
  f.cap->qp[par] = q;
  f.cap->recode[par] = q != qp;
}

int launch_size_cap(const FrameCtx& f, cudaStream_t st) {
  int n = launch_cavlc(f, st);
  k_size_cap<<<1, CAP_THREADS, 0, st>>>(f);
  n += 1 + launch_requant(f, st);
  return n + launch_cavlc_recode(f, st);
}

}  // namespace b2v
