// Legacy (mma.sync) tensor-pipe issue rates on this GPU: how many HMMA.16816 / IMMA.16832 an SM retires per cycle.
// The few-token contraction (qgemv.cu) spends one MMA per 256 (fp16) or 512 (int8) weights whatever the token
// count, so this rate, not HBM, can be the ceiling.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/mma_rate tools/mma_rate.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

template <int KIND>
__global__ void rate_kernel(int iters, uint32_t seed, float* out, long long* cycles) {
  uint32_t a[4] = {seed, seed ^ 1u, seed ^ 2u, seed ^ 3u}, b[2] = {seed ^ 5u, seed ^ 7u};
  float f[4][4] = {};
  int d[4][4] = {};
  uint32_t h[4][2] = {};
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      if (KIND == 0)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(f[c][0]), "+f"(f[c][1]), "+f"(f[c][2]), "+f"(f[c][3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
      else if (KIND == 1)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f16.f16.f16.f16 {%0,%1}, {%2,%3,%4,%5}, {%6,%7}, {%0,%1};"
                     : "+r"(h[c][0]), "+r"(h[c][1])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
      else if (KIND == 2)
        asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+r"(d[c][0]), "+r"(d[c][1]), "+r"(d[c][2]), "+r"(d[c][3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
      else if (KIND == 3)
        asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                     : "+f"(f[c][0]), "+f"(f[c][1]), "+f"(f[c][2]), "+f"(f[c][3])
                     : "r"(a[0]), "r"(a[1]), "r"(b[0]));
      else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(f[c][0]), "+f"(f[c][1]), "+f"(f[c][2]), "+f"(f[c][3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    }
  }
  long long t1 = clock64();
  float s = 0.f;
  for (int c = 0; c < 4; ++c)
    for (int j = 0; j < 4; ++j) s += f[c][j] + (float)d[c][j] + (float)h[c][j & 1];
  if (s == 123.456f) out[0] = s;
  if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int KIND>
void run(const char* name, int sms) {
  float* out;
  long long* cyc;
  cudaMalloc(&out, 4);
  cudaMalloc(&cyc, sizeof(long long) * sms);
  const int iters = 4096;
  for (int warps : {4, 8, 16, 32}) {
    rate_kernel<KIND><<<sms, warps * 32>>>(iters, 1u, out, cyc);
    rate_kernel<KIND><<<sms, warps * 32>>>(iters, 1u, out, cyc);
    cudaDeviceSynchronize();
    long long h[512];
    cudaMemcpy(h, cyc, sizeof(long long) * sms, cudaMemcpyDeviceToHost);
    double avg = 0;
    for (int i = 0; i < sms; ++i) avg += (double)h[i];
    avg /= sms;
    double per_sm_per_cycle = (double)warps * iters * 4 / avg;
    printf("{\"mma\": \"%s\", \"warps_per_sm\": %d, \"mma_per_cycle_per_sm\": %.4f, \"cycles_per_mma_per_smsp\": %.2f}\n", name,
           warps, per_sm_per_cycle, 4.0 / per_sm_per_cycle);
  }
  cudaFree(out);
  cudaFree(cyc);
}

int main() {
  cudaDeviceProp p;
  cudaGetDeviceProperties(&p, 0);
  int sms = p.multiProcessorCount;
  run<0>("m16n8k16.f32.f16", sms);
  run<1>("m16n8k16.f16.f16", sms);
  run<2>("m16n8k32.s32.s8", sms);
  run<3>("m16n8k8.f32.f16", sms);
  run<4>("m16n8k16.f32.bf16", sms);
  return 0;
}
