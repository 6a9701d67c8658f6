// read_lab.cu — what does a pure 33 MB read cost on this GPU?  (floor for the CSC kernel's input side)
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o tools/lab/read_lab tools/lab/read_lab.cu
#include <cstdio>
#include <cstdint>
#include <vector>
#include <algorithm>

__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
template <int U>
__global__ void k_read(const uint4* __restrict__ src, size_t n16, unsigned* sink, unsigned long long* ts) {
  if (threadIdx.x == 0 && ts) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMin(ts, t); }
  unsigned acc = 0;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < n16; i += U * stride) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++) v[u] = ldg_stream(src + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; u++) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
  }
  for (; i < n16; i += stride) { uint4 v = ldg_stream(src + i); acc ^= v.x ^ v.y ^ v.z ^ v.w; }
  if (acc == 0x12345678u) sink[0] = acc;
  if (ts) { __syncthreads(); if (threadIdx.x == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMax(ts + 1, t); } }
}
// read + write 3/8 as much (NV12-like) to a small L2-resident buffer
template <int U>
__global__ void k_read_write(const uint4* __restrict__ src, size_t n16, uint2* dst, unsigned long long* ts) {
  if (threadIdx.x == 0 && ts) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMin(ts, t); }
  size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < n16; i += U * stride) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++) v[u] = ldg_stream(src + i + u * stride);
#pragma unroll
    for (int u = 0; u < U; u++) dst[i + u * stride] = make_uint2(v[u].x ^ v[u].z, v[u].y ^ v[u].w);   // 8 B per 16 B read (a bit more than NV12's 6)
  }
  if (ts) { __syncthreads(); if (threadIdx.x == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMax(ts + 1, t); } }
}

int main() {
  const size_t fb = (size_t)3840 * 2160 * 4; const int NF = 8;
  std::vector<uint4*> in(NF);
  for (int i = 0; i < NF; i++) { cudaMalloc(&in[i], fb); cudaMemset(in[i], i + 1, fb); }
  unsigned* sink; cudaMalloc(&sink, 64);
  uint2* dst; cudaMalloc(&dst, fb / 2);
  unsigned long long* ts; cudaMalloc(&ts, 16);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  auto run = [&](const char* name, auto launch) {
    for (int i = 0; i < NF; i++) launch(i, nullptr);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    for (int i = 0; i < 200; i++) launch(i % NF, nullptr);
    cudaEventRecord(e1); cudaDeviceSynchronize();
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    double span = 0;
    for (int r = 0; r < 16; r++) {
      unsigned long long h[2] = {~0ull, 0}; cudaMemcpy(ts, h, 16, cudaMemcpyHostToDevice);
      launch(r % NF, ts); cudaDeviceSynchronize();
      cudaMemcpy(h, ts, 16, cudaMemcpyDeviceToHost); span += (h[1] - h[0]) * 1e-3;
    }
    printf("%-28s burst %.2f us/launch (%.0f GB/s read)   in-kernel span %.2f us (%.0f GB/s)  %s\n", name, ms * 1e3 / 200, fb / (ms * 1e-3 / 200) * 1e-9, span / 16, fb / (span / 16 * 1e-6) * 1e-9, cudaGetErrorString(cudaGetLastError()));
  };
  const size_t n16 = fb / 16;
  int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int ctas : {sms, 2 * sms, 4 * sms, 8 * sms, 16 * sms}) {
    char nm[64];
    snprintf(nm, 64, "read U4 %d x 256", ctas); run(nm, [&](int i, unsigned long long* t) { k_read<4><<<ctas, 256>>>(in[i], n16, sink, t); });
    snprintf(nm, 64, "read U8 %d x 256", ctas); run(nm, [&](int i, unsigned long long* t) { k_read<8><<<ctas, 256>>>(in[i], n16, sink, t); });
  }
  for (int ctas : {2 * sms, 4 * sms, 8 * sms}) {
    char nm[64];
    snprintf(nm, 64, "read U8 %d x 512", ctas); run(nm, [&](int i, unsigned long long* t) { k_read<8><<<ctas, 512>>>(in[i], n16, sink, t); });
    snprintf(nm, 64, "read+write U4 %d x 256", ctas); run(nm, [&](int i, unsigned long long* t) { k_read_write<4><<<ctas, 256>>>(in[i], n16, dst, t); });
  }
  // one-shot: one uint4 x U per thread
  run("read one-shot U4 (8100 CTAs)", [&](int i, unsigned long long* t) { k_read<4><<<(unsigned)(n16 / 4 / 256), 256>>>(in[i], n16, sink, t); });
  run("read one-shot U2 (16200 CTAs)", [&](int i, unsigned long long* t) { k_read<2><<<(unsigned)(n16 / 2 / 256), 256>>>(in[i], n16, sink, t); });
  return 0;
}
