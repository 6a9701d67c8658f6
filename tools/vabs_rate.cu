// micro-benchmark: issue rate of VABSDIFF4.U8.ACC (and IADD3 for reference) per SM on sm_90a (H100)
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/vabs_rate tools/vabs_rate.cu
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ unsigned sad4acc(unsigned a, unsigned b, unsigned c){ unsigned d; asm volatile("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
template<int MODE> __global__ void k(unsigned* out, int iters){
  unsigned a0=threadIdx.x, a1=a0*3+1, a2=a0*5+2, a3=a0*7+3, a4=a0*11, a5=a0*13, a6=a0*17, a7=a0*19, b=blockIdx.x*2654435761u;
  for(int i=0;i<iters;i++){
    if (MODE==0){ a0=sad4acc(a0,b,a0); a1=sad4acc(a1,b,a1); a2=sad4acc(a2,b,a2); a3=sad4acc(a3,b,a3); a4=sad4acc(a4,b,a4); a5=sad4acc(a5,b,a5); a6=sad4acc(a6,b,a6); a7=sad4acc(a7,b,a7);}
    else { asm volatile("add.u32 %0,%0,%1;":"+r"(a0):"r"(b)); asm volatile("add.u32 %0,%0,%1;":"+r"(a1):"r"(b)); asm volatile("add.u32 %0,%0,%1;":"+r"(a2):"r"(b)); asm volatile("add.u32 %0,%0,%1;":"+r"(a3):"r"(b));
           asm volatile("add.u32 %0,%0,%1;":"+r"(a4):"r"(b)); asm volatile("add.u32 %0,%0,%1;":"+r"(a5):"r"(b)); asm volatile("add.u32 %0,%0,%1;":"+r"(a6):"r"(b)); asm volatile("add.u32 %0,%0,%1;":"+r"(a7):"r"(b)); }
  }
  out[blockIdx.x*blockDim.x+threadIdx.x]=a0+a1+a2+a3+a4+a5+a6+a7;
}
int main(){
  cudaDeviceProp p; cudaGetDeviceProperties(&p,0);
  const int sms = p.multiProcessorCount;
  unsigned* d; cudaMalloc(&d, (size_t)sms*8*1024*4);
  for(int mode=0;mode<2;mode++){
    int iters=20000; dim3 g(sms*2), b(1024);
    cudaEvent_t e0,e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    if(mode==0) k<0><<<g,b>>>(d,100); else k<1><<<g,b>>>(d,100);
    cudaEventRecord(e0); if(mode==0) k<0><<<g,b>>>(d,iters); else k<1><<<g,b>>>(d,iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms,e0,e1);
    double winst = (double)g.x*b.x/32*iters*8;
    double per_sm_clk = winst/ (ms*1e-3) / sms / (p.clockRate*1e3);
    printf("%s: %.3f ms, %.2f warp-instr/clk/SM (clock %d kHz) => %.1f lanes/clk/SMSP\n", mode==0?"VABSDIFF4.ACC":"IADD", ms, per_sm_clk, p.clockRate, per_sm_clk*32/4);
  }
  return 0;
}
