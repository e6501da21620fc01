// p2p_store_bench.cu — how fast can ONE H100 store an index run into a peer GPU's HBM over NVLink,
// as a function of store width, CTAs and bytes in flight?  Decides the shape of gdv_sel_push
// (csrc/device/static_kernels.cu).  Single process, two devices, peer access enabled.
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a tools/p2p_store_bench.cu -o tools/_bin/p2p_store_bench
//   ./tools/_bin/p2p_store_bench          (on a machine with two GPUs)
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("%s failed: %s\n", #x, cudaGetErrorString(e)); exit(1); } } while (0)

template <typename T, int U>
__global__ void copy_strided(const T* __restrict__ src, T* dst, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < n; i += U * stride) {
    T v[U];
#pragma unroll
    for (int k = 0; k < U; ++k) v[k] = __ldcs(src + i + k * stride);
#pragma unroll
    for (int k = 0; k < U; ++k) dst[i + k * stride] = v[k];
  }
  for (; i < n; i += stride) dst[i] = src[i];
}

int main() {
  int nd = 0;
  CK(cudaGetDeviceCount(&nd));
  if (nd < 2) { printf("need 2 GPUs\n"); return 0; }
  const size_t bytes = 145ull << 20;
  void *src, *dst_peer, *dst_local;
  CK(cudaSetDevice(0));
  CK(cudaMalloc(&dst_peer, bytes + 256));
  CK(cudaSetDevice(1));
  CK(cudaDeviceEnablePeerAccess(0, 0));
  CK(cudaMalloc(&src, bytes));
  CK(cudaMalloc(&dst_local, bytes + 256));
  CK(cudaMemset(src, 1, bytes));
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  auto run = [&](const char* name, auto launch) {
    for (int peer = 0; peer < 2; ++peer) {
      void* d = peer ? (char*)dst_peer + 8 : (char*)dst_local + 8;   // 8-byte aligned, not 16: like a run at an odd offset
      for (int w = 0; w < 2; ++w) launch(d);
      CK(cudaEventRecord(e0));
      for (int r = 0; r < 5; ++r) launch(d);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      float ms;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("%-44s %s  %7.3f ms  %7.1f GB/s\n", name, peer ? "peer " : "local", ms / 5, bytes / (ms / 5) / 1e6);
    }
  };
  char name[128];
  // cudaMemcpyPeer reference (copy engine)
  {
    for (int w = 0; w < 2; ++w) CK(cudaMemcpyPeerAsync(dst_peer, 0, src, 1, bytes));
    CK(cudaEventRecord(e0));
    for (int r = 0; r < 5; ++r) CK(cudaMemcpyPeerAsync(dst_peer, 0, src, 1, bytes));
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    printf("%-44s peer   %7.3f ms  %7.1f GB/s\n", "cudaMemcpyPeerAsync (copy engine)", ms / 5, bytes / (ms / 5) / 1e6);
  }
  const int ctas_list[] = {4, 8, 16, 32, 132, 264};
  for (int ctas : ctas_list) {
    for (int bt : {256, 1024}) {
      snprintf(name, sizeof(name), "u64 x8 strided, %3d CTAs x %4d", ctas, bt);
      run(name, [&](void* d) { copy_strided<unsigned long long, 8><<<ctas, bt>>>((const unsigned long long*)src, (unsigned long long*)d, bytes / 8 - 2); });
      snprintf(name, sizeof(name), "ulonglong2 x4 strided, %3d CTAs x %4d", ctas, bt);
      // 16-byte stores need a 16-byte aligned destination: start one element later
      run(name, [&](void* d) { copy_strided<ulonglong2, 4><<<ctas, bt>>>((const ulonglong2*)src, (ulonglong2*)((char*)d + 8), bytes / 16 - 2); });
      snprintf(name, sizeof(name), "ulonglong2 x8 strided, %3d CTAs x %4d", ctas, bt);
      run(name, [&](void* d) { copy_strided<ulonglong2, 8><<<ctas, bt>>>((const ulonglong2*)src, (ulonglong2*)((char*)d + 8), bytes / 16 - 2); });
    }
  }
  return 0;
}
