// Read-only streaming bandwidth on this GPU: the denominator a weight-streaming kernel (qgemv.cu) can actually
// reach, as opposed to the copy figure (read + write) of MEASURED_PEAKS.json.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/read_bw tools/read_bw.cu
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

__global__ void read_ldg(const uint4* __restrict__ p, size_t n16, unsigned* out) {
  unsigned acc = 0;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  for (; i + 3 * stride < n16; i += 4 * stride) {
    uint4 a, b, c, d;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p + i));
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(p + i + stride));
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(c.x), "=r"(c.y), "=r"(c.z), "=r"(c.w) : "l"(p + i + 2 * stride));
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w) : "l"(p + i + 3 * stride));
    acc ^= a.x ^ a.y ^ a.z ^ a.w ^ b.x ^ b.y ^ b.z ^ b.w ^ c.x ^ c.y ^ c.z ^ c.w ^ d.x ^ d.y ^ d.z ^ d.w;
  }
  if (acc == 0x12345678u) out[0] = acc;
}

// one elected thread per CTA streams 16-KiB pieces with cp.async.bulk into a shared-memory ring; nobody reads them
__global__ void read_bulk(const unsigned char* __restrict__ p, size_t bytes, int stages) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + (size_t)stages * 16384);
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i)
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"((uint32_t)__cvta_generic_to_shared(&bar[i])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    size_t npieces = bytes / 16384;
    uint32_t it = 0;
    for (size_t pc = blockIdx.x; pc < npieces; pc += gridDim.x, ++it) {
      int slot = it % stages;
      uint32_t ph = (it / stages) & 1u;
      uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar[slot]);
      if (it >= (uint32_t)stages) {          // wait for the previous use of this slot to land
        uint32_t done = 0;
        while (!done)
          asm volatile("{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\n\tselp.u32 %0, 1, 0, q;\n\t}"
                       : "=r"(done) : "r"(b), "r"(ph ^ 1u) : "memory");
      }
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(16384u) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"((uint32_t)__cvta_generic_to_shared(smem + (size_t)slot * 16384)), "l"(p + pc * 16384), "r"(16384u), "r"(b) : "memory");
    }
    // drain
    for (int s = 0; s < stages && s < (int)it; ++s) {
      uint32_t i2 = it - 1 - s;
      uint32_t b = (uint32_t)__cvta_generic_to_shared(&bar[i2 % stages]);
      uint32_t done = 0;
      while (!done)
        asm volatile("{\n\t.reg .pred q;\n\tmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\n\tselp.u32 %0, 1, 0, q;\n\t}"
                     : "=r"(done) : "r"(b), "r"((i2 / stages) & 1u) : "memory");
    }
  }
}

int main() {
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  const int sms = prop.multiProcessorCount;
  const size_t bytes = (size_t)360 << 20;
  unsigned char *a, *b;
  unsigned* out;
  cudaMalloc(&a, bytes); cudaMalloc(&b, bytes); cudaMalloc(&out, 4);
  cudaMemset(a, 1, bytes); cudaMemset(b, 2, bytes);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int ctas_per_sm : {2, 4, 8}) {
    for (int rep = 0; rep < 2; ++rep) read_ldg<<<sms * ctas_per_sm, 512>>>((const uint4*)(rep ? b : a), bytes / 16, out);
    cudaEventRecord(e0);
    const int iters = 10;
    for (int i = 0; i < iters; ++i) read_ldg<<<sms * ctas_per_sm, 512>>>((const uint4*)((i & 1) ? b : a), bytes / 16, out);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("{\"kernel\": \"ldg128\", \"ctas_per_sm\": %d, \"GBps\": %.1f}\n", ctas_per_sm, bytes * iters / (ms / 1e3) / 1e9);
  }
  for (int stages : {4, 8, 12}) {
    size_t smem = (size_t)stages * 16384 + 256;
    cudaFuncSetAttribute(read_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    for (int rep = 0; rep < 2; ++rep) read_bulk<<<sms, 32, smem>>>(rep ? b : a, bytes, stages);
    cudaEventRecord(e0);
    const int iters = 10;
    for (int i = 0; i < iters; ++i) read_bulk<<<sms, 32, smem>>>((i & 1) ? b : a, bytes, stages);
    cudaEventRecord(e1); cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("{\"kernel\": \"cp.async.bulk 16KiB, 1 CTA/SM\", \"stages\": %d, \"GBps\": %.1f}\n", stages, bytes * iters / (ms / 1e3) / 1e9);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
