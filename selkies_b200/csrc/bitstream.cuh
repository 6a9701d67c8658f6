// bitstream.cuh — what the H.264 and JPEG encoders share between their entropy coders and their access units: the bit sinks the
// coders write through, and the block-wide routines that turn a word-packed bit string into escaped bytes (H.264 emulation
// prevention, 7.4.1; JPEG byte stuffing, T.81 F.1.2.3).
#pragma once
#include <climits>
#include <stdint.h>

namespace b2v {

// ------------------------------------------------------------------------------------------------ bit sinks
// A coder is a template over its sink: it runs once into a CountSink to size what it writes, once into a BitWriter to write it.
struct CountSink {
  int n = 0;
  __device__ __forceinline__ void put(int len, uint32_t) { n += len; }
};

// MSB-first into big-endian u32 words; writers that share words (neighbouring codes of other threads) meet in atomicOr.  The
// caller keeps v < 2^len.  Bits at or past `cap` are dropped while `pos` still advances, so a caller sees an overflow in `pos`.
struct BitWriter {
  uint32_t* w; long long pos; long long cap = LLONG_MAX;
  __device__ __forceinline__ void put(int len, uint32_t v) {
    if (len == 0) return;
    if (pos + len <= cap) {
      const long long wi = pos >> 5; const int o = (int)(pos & 31), space = 32 - o;
      if (len <= space) atomicOr(&w[wi], v << (space - len));
      else { atomicOr(&w[wi], v >> (len - space)); atomicOr(&w[wi + 1], v << (32 - (len - space))); }
    }
    pos += len;
  }
};

// byte i of a word-packed stream, read through L2 (see the block-wide routines below)
__device__ __forceinline__ uint32_t stream_byte(const uint32_t* w, long long i) { return (__ldcg(&w[i >> 2]) >> (24 - 8 * (int)(i & 3))) & 255u; }

// ------------------------------------------------------------------------------------------------ escape rules
// lead(w, i0): the rule's state in front of byte i0; take(state, b): does byte b take an escape byte (and advance the state)?
// `after`: the escape byte goes behind the byte (else in front of it); `byte`: its value.

// H.264 emulation prevention (7.4.1): a 0x03 goes in front of byte i when byte i <= 3 and the zero run in front of it is even
// and >= 2.  State: that zero run, which may begin before the bytes a thread reads.
struct H264Escape {
  static constexpr bool after = false; static constexpr uint8_t byte = 0x03;
  __device__ __forceinline__ static int lead(const uint32_t* w, long long i0) {
    int z = 0;
    while (i0 - 1 - z >= 0 && stream_byte(w, i0 - 1 - z) == 0u) z++;
    return z;
  }
  __device__ __forceinline__ static bool take(int& z, uint32_t b) { const bool e = b <= 3u && z >= 2 && (z & 1) == 0; z = b == 0u ? z + 1 : 0; return e; }
};

// JPEG byte stuffing (T.81 F.1.2.3): a 0x00 goes behind every 0xFF of the entropy-coded data.
struct JpegEscape {
  static constexpr bool after = true; static constexpr uint8_t byte = 0x00;
  __device__ __forceinline__ static int lead(const uint32_t*, long long) { return 0; }
  __device__ __forceinline__ static bool take(int&, uint32_t b) { return b == 255u; }
};

// ------------------------------------------------------------------------------------------------ block-wide routines
// For blocks of ESC_THREADS threads, every thread calling (they synchronise the block).  `scratch` is the caller's shared memory,
// ESC_THREADS / 32 ints that no thread still reads when the routine starts.  The segment is read through L2 (__ldcg), which is a
// matter of correctness: the count of k_slice_build reads words other blocks of the same launch wrote with atomicOr, the count of
// k_jpeg_ff reads the word thread 0 has just padded.
constexpr int ESC_THREADS = 256;

// byte offset of segment s in a sequence of segments: the sum of the sizes in front of it.  Every warp sums them itself, so the
// result needs no shared memory and no barrier.
__device__ __forceinline__ long long segment_offset(const uint32_t* size, int s) {
  long long t = 0;
  for (int j = threadIdx.x & 31; j < s; j += 32) t += size[j];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) t += __shfl_xor_sync(0xffffffffu, t, d);
  return t;
}

// words of bytes i0 .. i0 + 4 * NW - 1 of the stream (i0 a multiple of 4) into wd; returns the mask of the bytes below n that take
// an escape byte
template <class Rule, int NW>
__device__ __forceinline__ uint32_t escape_chunk(const uint32_t* w, long long i0, long long n, uint32_t (&wd)[NW]) {
  uint32_t mask = 0;
  int st = Rule::lead(w, i0);
#pragma unroll
  for (int k = 0; k < NW; k++) {
    wd[k] = i0 + 4 * k < n ? __ldcg(&w[(i0 + 4 * k) >> 2]) : 0u;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const uint32_t b = (wd[k] >> (24 - 8 * j)) & 255u;
      if (i0 + 4 * k + j < n && Rule::take(st, b)) mask |= 1u << (4 * k + j);
    }
  }
  return mask;
}

// escape bytes the n bytes of the word-packed segment w need, returned to every thread (one word per thread and round)
template <class Rule>
__device__ __forceinline__ int count_escapes(const uint32_t* w, long long n, int* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int cnt = 0;
  for (long long i0 = (long long)threadIdx.x * 4; i0 < n; i0 += ESC_THREADS * 4) { uint32_t wd[1]; cnt += __popc(escape_chunk<Rule>(w, i0, n, wd)); }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  if (lane == 0) scratch[warp] = cnt;
  __syncthreads();
  int t = 0;
#pragma unroll
  for (int ww = 0; ww < ESC_THREADS / 32; ww++) t += scratch[ww];
  return t;
}

// Copies the n bytes of the word-packed segment w, escaped, to out[o0 ...]; bytes at or past `cap` are dropped (the caller reports
// the overflow).  Then clears the segment's words (up to `words`) for the next picture, whose bits are again written with atomicOr.
// Returns the number of escape bytes written: the segment takes n + that many bytes of out.
template <class Rule>
__device__ __forceinline__ int copy_escaped(uint32_t* w, long long n, long long words, uint8_t* out, long long o0, long long cap, int* scratch) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int carry = 0;                                   // escape bytes of the rounds before
  constexpr int CH = 16;                           // bytes per thread and round
  for (long long cb = 0; cb < n; cb += (long long)ESC_THREADS * CH) {
    const long long i0 = cb + (long long)tid * CH;
    uint32_t wd[CH / 4];
    const uint32_t mask = i0 < n ? escape_chunk<Rule>(w, i0, n, wd) : 0u;
    const int cnt = __popc(mask);
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += o; }
    if (lane == 31) scratch[warp] = incl;
    __syncthreads();
    int before = carry + incl - cnt;
#pragma unroll
    for (int ww = 0; ww < ESC_THREADS / 32; ww++) { const int v = scratch[ww]; if (ww < warp) before += v; carry += v; }
    if (i0 < n) {
      long long o = o0 + i0 + before;
#pragma unroll
      for (int k = 0; k < CH; k++) {
        if (i0 + k < n) {
          const bool e = (mask >> k) & 1u;
          if (!Rule::after && e) { if (o < cap) out[o] = Rule::byte; o++; }
          if (o < cap) out[o] = (uint8_t)(wd[k >> 2] >> (24 - 8 * (k & 3)));
          o++;
          if (Rule::after && e) { if (o < cap) out[o] = Rule::byte; o++; }
        }
      }
    }
    __syncthreads();
  }
  const long long nw = min(words, (n >> 2) + 2);
  for (long long i = tid; i < nw; i += ESC_THREADS) w[i] = 0;
  return carry;
}

}  // namespace b2v
