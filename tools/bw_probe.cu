// Bandwidth probe for the BatchNorm-backward access pattern (2 streams in, 1 out, 16 B per thread-access).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/bw_probe tools/bw_probe.cu && /tmp/bw_probe
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdio>
#include <cstdint>

__device__ __forceinline__ uint4 ldg_stream(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ float silu_grad(float u, float d) {
  const float sg = __fdividef(1.f, 1.f + __expf(-u));
  return d * sg * (1.f + u * (1.f - sg));
}
__device__ __forceinline__ float blo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bhi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pk(float a, float b) { __nv_bfloat162 v = __floats2bfloat162_rn(a, b); return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ float2 h2f(uint32_t u) { __half2 h; *reinterpret_cast<uint32_t*>(&h) = u; return __half22float2(h); }

// MODE 0: pure copy-add (no math), MODE 1: full BN-backward math.  Linear indexing: vector i = blockIdx * (threads*ITERS) + ...
template <int U, int ITERS, int MODE, bool STREAM>
__global__ void __launch_bounds__(256) probe(const uint4* __restrict__ z, const uint4* __restrict__ d, uint4* __restrict__ o, size_t nvec,
                                              const float* __restrict__ cst, int cv) {
  const size_t base = static_cast<size_t>(blockIdx.x) * (256 * ITERS) + threadIdx.x;
  const int c8 = (threadIdx.x % cv) * 8;
  float s[8], t[8], A[8], B[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { s[k] = cst[c8 + k]; t[k] = cst[1024 + c8 + k]; A[k] = cst[2048 + c8 + k]; B[k] = cst[3072 + c8 + k]; }
#pragma unroll 1
  for (int it0 = 0; it0 < ITERS; it0 += U) {
    uint4 zq[U], dq[U];
    size_t idx[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      size_t i = base + static_cast<size_t>(it0 + u) * 256;
      idx[u] = i < nvec ? i : nvec - 1;
      if (STREAM) { zq[u] = ldg_stream(z + idx[u]); dq[u] = ldg_stream(d + idx[u]); }
      else { zq[u] = z[idx[u]]; dq[u] = d[idx[u]]; }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      uint4 r;
      if (MODE == 0) {
        r = make_uint4(zq[u].x ^ dq[u].x, zq[u].y ^ dq[u].y, zq[u].z ^ dq[u].z, zq[u].w ^ dq[u].w);
      } else {
        float zf[8], df[8], of[8];
        float2 a = h2f(zq[u].x), b = h2f(zq[u].y), c = h2f(zq[u].z), e = h2f(zq[u].w);
        zf[0] = a.x; zf[1] = a.y; zf[2] = b.x; zf[3] = b.y; zf[4] = c.x; zf[5] = c.y; zf[6] = e.x; zf[7] = e.y;
        df[0] = blo(dq[u].x); df[1] = bhi(dq[u].x); df[2] = blo(dq[u].y); df[3] = bhi(dq[u].y);
        df[4] = blo(dq[u].z); df[5] = bhi(dq[u].z); df[6] = blo(dq[u].w); df[7] = bhi(dq[u].w);
#pragma unroll
        for (int k = 0; k < 8; ++k) of[k] = fmaf(s[k], silu_grad(fmaf(zf[k], s[k], t[k]), df[k]), fmaf(A[k], zf[k], B[k]));
        r = make_uint4(pk(of[0], of[1]), pk(of[2], of[3]), pk(of[4], of[5]), pk(of[6], of[7]));
      }
      if (base + static_cast<size_t>(it0 + u) * 256 < nvec) o[idx[u]] = r;
    }
  }
}

template <int U, int ITERS, int MODE, bool STREAM>
void run(const char* name, const uint4* z, const uint4* d, uint4* o, size_t nvec, const float* cst, int cv) {
  const unsigned grid = static_cast<unsigned>((nvec + 256 * ITERS - 1) / (256 * ITERS));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 2; ++i) probe<U, ITERS, MODE, STREAM><<<grid, 256>>>(z, d, o, nvec, cst, cv);
  cudaEventRecord(e0);
  const int reps = 5;
  for (int i = 0; i < reps; ++i) probe<U, ITERS, MODE, STREAM><<<grid, 256>>>(z, d, o, nvec, cst, cv);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, probe<U, ITERS, MODE, STREAM>, 256, 0);
  cudaFuncAttributes fa; cudaFuncGetAttributes(&fa, probe<U, ITERS, MODE, STREAM>);
  printf("%-34s U=%d iters=%2d regs=%3d blocks/SM=%d  %8.1f us  %7.1f GB/s\n", name, U, ITERS, fa.numRegs, occ, 1e3 * ms / reps,
         nvec * 48.0 / (ms / reps * 1e-3) / 1e9);
}

int main() {
  const size_t nvec = 6553600ull * 4;  // stem layer: 6.5 M pixels x 32 channels = 210 M elements (1.26 GB of traffic)
  uint4 *z, *d, *o; float* cst;
  cudaMalloc(&z, nvec * 16); cudaMalloc(&d, nvec * 16); cudaMalloc(&o, nvec * 16); cudaMalloc(&cst, 4096 * 4);
  cudaMemset(z, 0x11, nvec * 16); cudaMemset(d, 0x22, nvec * 16); cudaMemset(cst, 0, 4096 * 4);
  run<1, 8, 0, false>("copy  plain", z, d, o, nvec, cst, 4);
  run<2, 8, 0, false>("copy  plain", z, d, o, nvec, cst, 4);
  run<4, 8, 0, false>("copy  plain", z, d, o, nvec, cst, 4);
  run<4, 8, 0, true>("copy  L1::no_allocate", z, d, o, nvec, cst, 4);
  run<8, 8, 0, true>("copy  L1::no_allocate", z, d, o, nvec, cst, 4);
  run<4, 16, 0, true>("copy  L1::no_allocate", z, d, o, nvec, cst, 4);
  run<1, 8, 1, true>("bnbwd L1::no_allocate", z, d, o, nvec, cst, 4);
  run<2, 8, 1, true>("bnbwd L1::no_allocate", z, d, o, nvec, cst, 4);
  run<4, 8, 1, true>("bnbwd L1::no_allocate", z, d, o, nvec, cst, 4);
  run<2, 8, 1, false>("bnbwd plain", z, d, o, nvec, cst, 4);
  run<4, 16, 1, true>("bnbwd L1::no_allocate", z, d, o, nvec, cst, 4);
  run<2, 2, 1, true>("bnbwd L1::no_allocate", z, d, o, nvec, cst, 4);
  run<1, 1, 1, true>("bnbwd L1::no_allocate", z, d, o, nvec, cst, 4);
  cudaError_t e = cudaDeviceSynchronize();
  printf("status: %s\n", cudaGetErrorString(e));
  return 0;
}
