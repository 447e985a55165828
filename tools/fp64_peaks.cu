// Microbenchmark: fp64 peaks of an H100 (sm_90a) -- DFMA, DMMA.8x8x4, exp().
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_peaks fp64_peaks.cu
// Output: one JSON object on stdout (the source of the fp64 peaks bench.py divides by).
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){fprintf(stderr,"CUDA %s at %d\n",cudaGetErrorString(e),__LINE__); exit(1);} }while(0)

template<int ILP>
__global__ void dfma_kernel(double* out, double x, int iters){
  double acc[ILP];
  #pragma unroll
  for(int i=0;i<ILP;i++) acc[i]=threadIdx.x*1e-9+i;
  double m = x;
  for(int it=0; it<iters; ++it){
    #pragma unroll
    for(int i=0;i<ILP;i++) acc[i]=fma(acc[i],m,1e-300);
  }
  double s=0;
  #pragma unroll
  for(int i=0;i<ILP;i++) s+=acc[i];
  if(s==123.456) out[0]=s;
}

template<int NACC>
__global__ void dmma_kernel(double* out, double x, int iters){
  double c0[NACC], c1[NACC];
  #pragma unroll
  for(int i=0;i<NACC;i++){ c0[i]=0; c1[i]=0; }
  double a = x*threadIdx.x, b = x+threadIdx.x;
  for(int it=0; it<iters; ++it){
    #pragma unroll
    for(int i=0;i<NACC;i++){
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1},{%2},{%3},{%0,%1};"
                   :"+d"(c0[i]),"+d"(c1[i]):"d"(a),"d"(b));
    }
  }
  double s=0;
  #pragma unroll
  for(int i=0;i<NACC;i++) s+=c0[i]+c1[i];
  if(s==123.456) out[0]=s;
}

// DMMA and DFMA issued together: do they share a pipe?
template<int NACC, int NF>
__global__ void mixed_kernel(double* out, double x, int iters){
  double c0[NACC], c1[NACC], f[NF>0?NF:1];
  #pragma unroll
  for(int i=0;i<NACC;i++){ c0[i]=0; c1[i]=0; }
  #pragma unroll
  for(int i=0;i<NF;i++) f[i]=i+threadIdx.x*1e-9;
  double a = x*threadIdx.x, b = x+threadIdx.x;
  for(int it=0; it<iters; ++it){
    #pragma unroll
    for(int i=0;i<NACC;i++){
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1},{%2},{%3},{%0,%1};"
                   :"+d"(c0[i]),"+d"(c1[i]):"d"(a),"d"(b));
    }
    #pragma unroll
    for(int i=0;i<NF;i++) f[i]=fma(f[i],x,1e-300);
  }
  double s=0;
  #pragma unroll
  for(int i=0;i<NACC;i++) s+=c0[i]+c1[i];
  #pragma unroll
  for(int i=0;i<NF;i++) s+=f[i];
  if(s==123.456) out[0]=s;
}

__global__ void exp_kernel(double* out, double x, int iters){
  double v0 = -1e-3*threadIdx.x - x, v1=v0*1.1, v2=v0*1.2, v3=v0*1.3;
  double s0=0,s1=0,s2=0,s3=0;
  for(int it=0; it<iters; ++it){
    s0+=exp(v0); s1+=exp(v1); s2+=exp(v2); s3+=exp(v3);
    v0-=1e-6; v1-=1e-6; v2-=1e-6; v3-=1e-6;
  }
  double s=s0+s1+s2+s3;
  if(s==123.456) out[0]=s;
}

template<class F>
float time_ms(F launch, int reps){
  cudaEvent_t e0,e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  launch(); launch(); CK(cudaDeviceSynchronize());
  float best=1e30f;
  for(int r=0;r<reps;r++){
    CK(cudaEventRecord(e0)); launch(); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
    float ms; CK(cudaEventElapsedTime(&ms,e0,e1)); if(ms<best) best=ms;
  }
  return best;
}

int main(){
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p,0));
  int sms=p.multiProcessorCount;
  double* out; CK(cudaMalloc(&out,8));
  printf("{\"gpu\":\"%s\",\"sms\":%d,\"clock_khz\":%d", p.name, sms, p.clockRate);
  const int iters=20000;
  // DFMA
  for(int warps : {4,8,16,32}){
    int thr=warps*32; int blocks=sms*1;
    float ms=time_ms([&]{dfma_kernel<8><<<blocks,thr>>>(out,1.0000001,iters);},5);
    double fl=2.0*8*iters*(double)thr*blocks;
    printf(",\"dfma_tflops_w%d\":%.3f",warps,fl/ms*1e-9);
  }
  // DMMA
  for(int warps : {4,8,16,32}){
    int thr=warps*32; int blocks=sms;
    float ms=time_ms([&]{dmma_kernel<8><<<blocks,thr>>>(out,1.0000001,iters);},5);
    double fl=2.0*256*8*iters*(double)warps*blocks;
    printf(",\"dmma_tflops_w%d_acc8\":%.3f",warps,fl/ms*1e-9);
  }
  for(int warps : {4,8,16}){
    int thr=warps*32; int blocks=sms;
    float ms=time_ms([&]{dmma_kernel<2><<<blocks,thr>>>(out,1.0000001,iters);},5);
    double fl=2.0*256*2*iters*(double)warps*blocks;
    printf(",\"dmma_tflops_w%d_acc2\":%.3f",warps,fl/ms*1e-9);
  }
  { // single warp per SM, dependent chain -> latency
    float ms=time_ms([&]{dmma_kernel<1><<<sms,32>>>(out,1.0000001,iters);},3);
    printf(",\"dmma_dep_latency_ns\":%.2f",ms*1e6/iters);
    float ms2=time_ms([&]{dfma_kernel<1><<<sms,32>>>(out,1.0000001,iters);},3);
    printf(",\"dfma_dep_latency_ns\":%.2f",ms2*1e6/iters);
  }
  // mixed: 8 DMMA (=2048 FMA) + NF*32 DFMA per warp-iteration
  {
    int warps=8, thr=256, blocks=sms;
    float m0=time_ms([&]{mixed_kernel<8,0><<<blocks,thr>>>(out,1.0000001,iters);},5);
    float m8=time_ms([&]{mixed_kernel<8,8><<<blocks,thr>>>(out,1.0000001,iters);},5);
    float m16=time_ms([&]{mixed_kernel<8,16><<<blocks,thr>>>(out,1.0000001,iters);},5);
    printf(",\"mixed_ms_dmma8_dfma0\":%.4f,\"mixed_ms_dmma8_dfma8\":%.4f,\"mixed_ms_dmma8_dfma16\":%.4f",m0,m8,m16);
    (void)warps;
  }
  // exp
  for(int warps : {8,16,32}){
    int thr=warps*32, blocks=sms; int it2=4000;
    float ms=time_ms([&]{exp_kernel<<<blocks,thr>>>(out,1.0,it2);},5);
    double n=4.0*it2*(double)thr*blocks;
    printf(",\"exp_gexp_per_s_w%d\":%.2f",warps,n/ms*1e-6);
  }
  printf("}\n");
  return 0;
}
